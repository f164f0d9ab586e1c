"""obs_intr_cols (theiasfm_b200/csrc/tba_camera_models.cuh) compiled for the host: under the TRIVIAL loss the intrinsics columns
rebuilt from the normalised image point (u, v) that linearize_obs reports are bit for bit the J_i it returns -- what the compact
layout of the stored linearisation relies on -- with and without FMA contraction by the compiler.  Under a robust loss J_i
carries the corrector and the identity rebuild differs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import golden_problem

HERE = os.path.dirname(os.path.abspath(__file__))
HDRS = [os.path.join(HERE, "..", "theiasfm_b200", "csrc", h) for h in ("tba_camera_models.cuh", "tba_camera_models_ext.cuh")]


def _lib(tag, flags):
    src = os.path.join(HERE, "host_intr_cols.cc")
    so = os.path.join(HERE, "_host_intr_cols_%s.so" % tag)
    if not os.path.exists(so) or max([os.path.getmtime(src)] + [os.path.getmtime(h) for h in HDRS]) > os.path.getmtime(so):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared"] + flags + ["-x", "c++", src, "-o", so])
    L = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    L.host_intr_cols.argtypes = [C.c_int, dp, dp, dp, dp, C.c_int, C.c_double, dp, dp, dp]
    return L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _observations():
    """the golden observations of both models, and the same with distortion and skew large enough to move every column"""
    prob, g = golden_problem()
    rng = np.random.default_rng(5)
    out = []
    for i in range(prob.n_obs):
        ext, intr, pt, xy = (np.ascontiguousarray(g[k][i], np.float64) for k in ("ext", "intr", "pt", "xy"))
        out.append((int(g["model"][i]), ext, intr, pt, xy))
        intr2 = intr.copy()
        intr2[1] *= 1.0 + 0.1 * rng.uniform(-1, 1)
        intr2[2] = 0.3 * rng.uniform(-1, 1)
        intr2[5:10] = 0.05 * rng.uniform(-1, 1, 5)
        out.append((int(g["model"][i]), ext, intr2, pt, xy))
    return out


@pytest.mark.parametrize("tag,flags", [("exact", ["-ffp-contract=off"]), ("fma", ["-mfma", "-ffp-contract=fast"])])
def test_rebuilt_intrinsics_columns_are_bit_identical_under_the_trivial_loss(tag, flags):
    L = _lib(tag, flags)
    n = 0
    for model, ext, intr, pt, xy in _observations():
        Ji, uv, Jr = np.zeros(20), np.zeros(2), np.zeros(20)
        if not L.host_intr_cols(model, _dp(ext), _dp(intr), _dp(pt), _dp(xy), 0, 1.0, _dp(Ji), _dp(uv), _dp(Jr)):
            continue
        n += 1
        assert np.isfinite(uv).all()
        assert np.array_equal(Ji.view(np.int64), Jr.view(np.int64)), (model, Ji, Jr)
        # a HUBER loss whose width no residual reaches is the same arithmetic
        Jh = np.zeros(20)
        assert L.host_intr_cols(model, _dp(ext), _dp(intr), _dp(pt), _dp(xy), 1, 1e30, _dp(Jh), _dp(uv), _dp(Jr)) == 1
        assert np.array_equal(Jh.view(np.int64), Ji.view(np.int64))
    assert n >= 4


def test_a_robust_corrector_is_not_the_identity_rebuild():
    L = _lib("exact", ["-ffp-contract=off"])
    model, ext, intr, pt, xy = _observations()[0]
    xy = xy + 30.0  # an outlier: the CAUCHY corrector scales and rotates the rows
    Ji, uv, Jr = np.zeros(20), np.zeros(2), np.zeros(20)
    assert L.host_intr_cols(model, _dp(ext), _dp(intr), _dp(pt), _dp(xy), 3, 1.0, _dp(Ji), _dp(uv), _dp(Jr)) == 1
    assert not np.allclose(Ji, Jr)
