"""BundleAdjustViewsB200 (adapter/bundle_adjust_views_b200.cc: batched BundleAdjustView through tba_adjust_views) end to end on a
GPU, against BundleAdjustView restated view after view with the oracle (tests/adapter_views_test.cc)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAPTER = os.path.join(ROOT, "adapter")


@pytest.fixture(scope="module")
def views_test_bin(oracle, request):
    if request.config.getoption("--mock-engine"):
        pytest.skip("binary driver: needs the real CUDA engine or its emulation build")
    if request.config.getoption("--emulate-engine"):  # the same driver and adapter, linked with the SIMT-emulated engine (tests/emu)
        emu = os.path.join(ROOT, "tests", "emu")
        out = os.path.join(ROOT, "tests", "adapter_views_test_emu")
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++14", "-fPIC", "-I" + os.path.join(ADAPTER, "theia_compat"), "-I" + os.path.join(ROOT, "include"),
                               "-I" + ADAPTER, "-o", out, os.path.join(ROOT, "tests", "adapter_views_test.cc"),
                               os.path.join(ADAPTER, "bundle_adjuster_b200.cc"), os.path.join(ADAPTER, "bundle_adjust_views_b200.cc"),
                               "-L" + emu, "-ltheia_ba_b200_emu", "-Wl,-rpath," + emu, "-ldl", "-lpthread"])
        return out
    subprocess.check_call(["make", "-C", ADAPTER], stdout=subprocess.DEVNULL)
    return os.path.join(ADAPTER, "adapter_views_test")


@pytest.mark.gpu
def test_bundle_adjust_views_against_oracle(views_test_bin):
    out = subprocess.run([views_test_bin, "views", os.path.join(ROOT, "oracle", "libba_oracle.so")], capture_output=True, text=True, timeout=1500)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "views ok" in out.stdout
