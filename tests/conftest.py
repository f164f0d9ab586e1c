import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_addoption(parser):
    parser.addoption("--emulate-engine", action="store_true", default=False,
                     help="run the -m gpu test files on the CPU through the REAL engine code compiled against the SIMT emulator of "
                          "tests/emu (control flow, indexing, reductions, host glue -- not performance)")
    parser.addoption("--mock-engine", action="store_true", default=False,
                     help="run the -m gpu test files on the CPU against tests/mock_engine_py.py (checks the TESTS, not the engine)")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu on a machine with an H100)")
    if config.getoption("--mock-engine"):
        import mock_engine_py
        mock_engine_py.install()
    if config.getoption("--emulate-engine"):
        import subprocess
        emu = os.path.join(ROOT, "tests", "emu")
        subprocess.check_call(["make", "-C", emu], stdout=subprocess.DEVNULL)
        from theiasfm_b200 import engine
        engine.LIB_PATH = os.path.join(emu, os.environ.get("TBA_EMU_LIBNAME", "libtheia_ba_b200_emu.so"))  # or the asan build, see tests/emu/Makefile
        engine._LIB = None
        from theiasfm_b200 import matcher
        matcher.LIB_PATH = os.path.join(emu, "libtheia_matcher_b200_emu.so")
        matcher._LIB = None
        # spawned rank processes (test_y_multi_gpu) inherit these: two emulated devices, shared-memory NCCL stand-in
        os.environ["THEIA_BA_B200_LIB"] = engine.LIB_PATH
        os.environ["TBA_EMU_NCCL"] = os.path.join(emu, "libemu_nccl.so")
        os.environ.setdefault("TBA_EMU_DEVICES", "2")


def pytest_collection_modifyitems(config, items):
    if not (config.getoption("--mock-engine") or config.getoption("--emulate-engine")):
        return
    skip = pytest.mark.skip(reason="needs the real CUDA engine or its emulation build (binary / multi-process / matcher library)")
    too_big = pytest.mark.skip(reason="full-size scene: hours under the SIMT emulator")
    emu_big = ("test_x_fullsize_gpu", "test_tensor_core_path_equals")
    for item in items:
        names = () if config.getoption("--emulate-engine") else ("test_xx_matcher_gpu", "test_z_adapter_gpu", "test_y_multi_gpu")
        if any(k in item.nodeid for k in names):
            item.add_marker(skip)
        elif config.getoption("--emulate-engine") and any(k in item.nodeid for k in emu_big):
            item.add_marker(too_big)


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle_py
    oracle_py.build()
    # the GPU boxes are shared hosts with 128 logical CPUs: a 128-thread OpenMP team there spends its time in barrier spins whenever
    # a neighbour is busy (a 20 s test file took 20 min in round 2); the checker does not need more than 32 threads
    oracle_py.set_num_threads(min(32, len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 8))
    return oracle_py
