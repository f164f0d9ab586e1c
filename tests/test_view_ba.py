"""N3 (SURVEY 8f): batched BundleAdjustView (bundle_adjustment.cc:83-93) on the CPU.

* tests/view_ba_oracle.py, the serial restatement the GPU tests compare against, agrees with the oracle's own solver
  (oracle_py.solve, DENSE_QR, no inner iterations) on the single-view sub-problem of every view;
* the product's per-view body (theiasfm_b200/csrc/tba_view_ba.cuh, one CTA per view in k_view_ba) compiled for the host agrees with
  the restatement, with one lane and as a 4-lane team of host threads;
* the refusals (shared free intrinsics group, bad indices) and the degenerate views."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import view_ba_oracle as vbo
from theiasfm_b200 import _abi

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def H():
    so, src = os.path.join(HERE, "_host_view_ba.so"), os.path.join(HERE, "host_view_ba.cc")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", src, "-o", so])
    L = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    L.host_view_ba.argtypes = [C.POINTER(_abi.tba_options), dp, dp, C.c_int, C.c_uint, C.c_int, dp, dp, C.c_int, dp]
    return L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def run_host(H, problem, options, cam, team):
    """The product body on view `cam` of problem (updated in place): (termination, initial, final, iterations)."""
    sel = np.nonzero(problem.obs_cam == cam)[0]
    g = int(problem.cam_group[cam])
    fm = vbo.free_mask(problem, cam)
    ext = problem.ext[cam].copy(); intr = problem.intr[g].copy()
    pt = np.ascontiguousarray(problem.pt[problem.obs_pt[sel]]); xy = np.ascontiguousarray(problem.obs_xy[sel])
    out = np.zeros(4)
    H.host_view_ba(C.byref(options), _dp(ext), _dp(intr), int(problem.group_model[g]), int(sum(1 << j for j in range(16) if fm[j])), len(sel),
                   _dp(pt), _dp(xy), int(team), _dp(out))
    problem.ext[cam] = ext; problem.intr[g] = intr
    return int(out[0]), out[1], out[2], int(out[3])


def rel(a, b):
    return 0.0 if a == b else abs(a - b) / abs(b)


@pytest.mark.parametrize("name", sorted(vbo.SCENES))
def test_restatement_matches_oracle_solve_per_view(oracle, name):
    p, kw = vbo.view_scene(name)
    o = oracle.default_options(**kw)
    n_moved = 0
    for cam in range(p.n_cam):
        q = p.copy()
        st, ic, fc, it = vbo.adjust_views(q, o, [cam])
        sub, _ = vbo.single_view_problem(p, cam)
        s = oracle.solve(sub, o)
        assert s.rc == 0
        assert st[0] == s.termination_type and it[0] == s.num_iterations - 1, (cam, st, it, s.termination_type, s.num_iterations, s.message)
        assert rel(ic[0], s.initial_cost) <= 1e-12 and rel(fc[0], s.final_cost) <= 1e-12
        assert np.allclose(q.ext[cam], sub.ext[0], rtol=1e-9, atol=1e-12)
        assert np.allclose(q.intr[p.cam_group[cam]], sub.intr[0], rtol=1e-9, atol=1e-12)
        n_moved += it[0] > 0 and fc[0] < 0.9 * ic[0]
    assert n_moved >= p.n_cam // 2


@pytest.mark.parametrize("name", sorted(vbo.SCENES))
@pytest.mark.parametrize("team", [False, True], ids=["serial", "team4"])
def test_host_body_matches_restatement(H, oracle, name, team):
    p, kw = vbo.view_scene(name, n_cam=8, n_pt=150)
    o = oracle.default_options(**kw)
    for cam in range(p.n_cam):
        q, h = p.copy(), p.copy()
        st, ic, fc, it = vbo.adjust_views(q, o, [cam])
        th, ich, fch, ith = run_host(H, h, o, cam, team)
        assert th == st[0] and ith == it[0], (cam, th, st[0], ith, it[0])
        assert rel(ich, ic[0]) <= 1e-11 and rel(fch, fc[0]) <= 1e-7
        g = p.cam_group[cam]
        assert np.abs(h.ext[cam] - q.ext[cam]).max() <= 1e-8 * np.abs(q.ext[cam]).max()
        assert np.abs(h.intr[g] - q.intr[g]).max() <= 1e-8 * np.abs(q.intr[g]).max()


def degenerate_scene():
    """Camera 0 has no observation, camera 1 no free coordinate, camera 2 sees a point at its own centre (the functor fails)."""
    p, kw = vbo.view_scene("radtan_per_camera_all", n_cam=8, n_pt=150)
    keep = p.obs_cam != 0
    p = _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const, p.obs_cam[keep],
                     p.obs_pt[keep], p.obs_xy[keep])
    p.ext_const[1] = _abi.EXT_ALL_CONST
    p.group_const_mask[p.cam_group[1]] = 0x3FF
    k = int(np.nonzero(p.obs_cam == 2)[0][0])
    p.pt[p.obs_pt[k]] = np.concatenate([p.ext[2, :3], [1.0]])
    return p, kw


def test_degenerate_views(H, oracle):
    p, kw = degenerate_scene()
    o = oracle.default_options(**kw)
    for cam, term in ((0, _abi.CONVERGENCE), (1, _abi.CONVERGENCE), (2, _abi.FAILURE)):
        sub, _ = vbo.single_view_problem(p, cam)
        s = oracle.solve(sub, o)
        q = p.copy()
        st, ic, fc, it = vbo.adjust_views(q, o, [cam])
        assert st[0] == term == s.termination_type and it[0] == 0 == s.num_iterations - (0 if term == _abi.FAILURE else 1)
        assert ic[0] == s.initial_cost and fc[0] == s.final_cost
        assert np.array_equal(q.ext, p.ext) and np.array_equal(q.intr, p.intr)
        for team in (False, True):
            h = p.copy()
            th, ich, fch, ith = run_host(H, h, o, cam, team)
            assert (th, ith) == (term, 0) and rel(ich, ic[0]) <= 1e-12 and rel(fch, fc[0]) <= 1e-12
            assert np.array_equal(h.ext, p.ext) and np.array_equal(h.intr, p.intr)
    # no observations: cost 0; no free coordinate: Ceres' fixed cost; failed functor: -1
    s0 = vbo.adjust_views(p.copy(), o, [0]); s1 = vbo.adjust_views(p.copy(), o, [1]); s2 = vbo.adjust_views(p.copy(), o, [2])
    assert s0[1][0] == 0.0 == s0[2][0] and s1[1][0] > 0.0 and s1[1][0] == s1[2][0] and s2[1][0] == -1.0 == s2[2][0]


def test_refusals():
    p, _ = vbo.view_scene("pinhole_shared_default", n_cam=6, n_pt=100)
    assert vbo.check_views(p, [0, 1]) == _abi.ERR_INVALID_ARGUMENT          # shared group with free focal length / radial
    assert vbo.check_views(p, [0]) == _abi.OK
    assert vbo.check_views(p, [0, 0]) == _abi.ERR_INVALID_ARGUMENT and vbo.check_views(p, [6]) == _abi.ERR_INVALID_ARGUMENT
    assert vbo.check_views(p, [-1]) == _abi.ERR_INVALID_ARGUMENT
    p.group_const_mask[:] = 0x3FF                                               # a fully constant shared group may be batched
    assert vbo.check_views(p, list(range(6))) == _abi.OK
    q, _ = vbo.view_scene("radtan_per_camera_all", n_cam=6, n_pt=100)
    assert vbo.check_views(q, list(range(6))) == _abi.OK
    with pytest.raises(ValueError):
        vbo.adjust_views(p.copy(), None, [1, 1])
    assert [len(b) for b in vbo.batches(vbo.view_scene("pinhole_shared_default", n_cam=6, n_pt=100)[0], range(6))] == [1] * 6
