"""The streaming kernels replace the key shuffles of the segmented warp reduction by a run structure derived from
the ballot of the run heads (theiasfm_b200/csrc/tba_segments.h).  Checked on the CPU: run_last_lane against brute force for random
run layouts (including the tile layouts the pack produces: points, then unique negative keys for padding lanes), and the two
reductions -- emulated with __shfl_down_sync's semantics -- give bit-identical results in every lane that starts a run."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def H():
    so, src = os.path.join(HERE, "_host_segments.so"), os.path.join(HERE, "host_segments.cc")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", src, "-o", so])
    return C.CDLL(so)


def layouts(rng, n):
    for _ in range(n):
        kind = rng.integers(0, 4)
        if kind == 0:      # random run lengths
            keys, k = [], 0
            while len(keys) < 32:
                keys += [k] * int(rng.integers(1, 12)); k += 1
            yield np.array(keys[:32], np.int32)
        elif kind == 1:    # a packed warp slice: points of 2..10 observations, then padding lanes with unique negative keys
            keys, k = [], 0
            while True:
                ln = int(rng.integers(2, 11))
                if len(keys) + ln > 32:
                    break
                keys += [k] * ln; k += 1
            keys += [-1 - l for l in range(len(keys), 32)]
            yield np.array(keys, np.int32)
        elif kind == 2:    # one run (a long track's warp)
            yield np.zeros(32, np.int32)
        else:              # every lane its own run
            yield np.arange(32, dtype=np.int32)


def test_run_last_lane_and_reduction_equivalence(H):
    rng = np.random.default_rng(5)
    for keys in layouts(rng, 400):
        heads = 0
        for l in range(32):
            if l == 0 or keys[l - 1] != keys[l]:
                heads |= 1 << l
        for l in range(32):
            want = l
            while want + 1 < 32 and keys[want + 1] == keys[l]:
                want += 1
            assert H.host_run_last_lane(C.c_uint(heads), l) == want
        vals = rng.normal(size=32) * 10.0 ** rng.integers(-3, 4, 32)
        a, b = np.zeros(32), np.zeros(32)
        dp = C.POINTER(C.c_double)
        H.host_seg_reduce_both(keys.ctypes.data_as(C.POINTER(C.c_int)), vals.ctypes.data_as(dp), a.ctypes.data_as(dp), b.ctypes.data_as(dp))
        assert np.array_equal(a, b)                      # every lane, bit for bit (same additions in the same order)
        for l in range(32):                              # and the run heads hold the run sums
            if l == 0 or keys[l - 1] != keys[l]:
                run = keys == keys[l]
                assert abs(a[l] - vals[run].sum()) <= 1e-12 * np.abs(vals[run]).sum()
