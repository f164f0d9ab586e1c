"""N3 on the GPU, through the C-ABI: tba_adjust_views (batched BundleAdjustView, one CTA per view, k_view_ba) on the
device-resident problem, against the serial restatement of tests/view_ba_oracle.py (itself checked against the oracle's solver by
tests/test_view_ba.py, which also runs the kernel's body on the host)."""
import numpy as np
import pytest

import view_ba_oracle as vbo
from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu
vbo.extend_mock_engine()


def rel_err(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.abs(a - b) / np.maximum(np.abs(b), 1e-300)


def run_engine(p, kw, views):
    """Batches of views on one upload; returns per-view results in view order and the downloaded problem."""
    q = p.copy()
    eng = engine.Engine()
    eng.upload(q, engine.default_options(**kw))
    out = [eng.adjust_views(engine.default_options(**kw), b) for b in vbo.batches(p, views)]
    eng.download(q)
    eng.close()
    return [np.concatenate(x) for x in zip(*out)], q


def run_oracle(p, kw, views, oracle):
    q = p.copy()
    o = oracle.default_options(**kw)
    out = [vbo.adjust_views(q, o, b) for b in vbo.batches(p, views)]
    return [np.concatenate(x) for x in zip(*out)], q


def compare(res_e, qe, res_o, qo, views, p):
    st, ic, fc, it = res_e
    so, ico, fco, ito = res_o
    assert np.array_equal(st, so) and np.array_equal(it, ito), (st, so, it, ito)
    ok = ico > 0
    assert (rel_err(ic[ok], ico[ok]) <= 1e-11).all()
    # a final cost at the rounding floor of the initial one (a view with fewer residuals than unknowns: the oracle ends below
    # 1e-6 of its initial cost) is compared to that floor; every other view at 1e-7 relative
    floor = np.where(fco[ok] < 1e-6 * ico[ok], 1e-12 * ico[ok], 0.0)
    assert (np.abs(fc[ok] - fco[ok]) <= np.maximum(1e-7 * fco[ok], floor)).all()
    assert np.array_equal(ic[~ok], ico[~ok]) and np.array_equal(fc[~ok], fco[~ok])
    assert np.abs(qe.ext - qo.ext).max() <= 1e-8 * np.abs(qo.ext).max()
    for g in range(p.n_group):
        assert np.abs(qe.intr[g] - qo.intr[g]).max() <= 1e-8 * np.abs(qo.intr[g]).max()
    # points never move; cameras outside the batch and constant coordinates come back bit-identical
    assert np.array_equal(qe.pt, p.pt)
    others = np.setdiff1d(np.arange(p.n_cam), views)
    assert np.array_equal(qe.ext[others], p.ext[others])
    pos_c = (p.ext_const & _abi.EXT_POSITION_CONST) != 0
    ori_c = (p.ext_const & _abi.EXT_ORIENTATION_CONST) != 0
    assert np.array_equal(qe.ext[pos_c, :3], p.ext[pos_c, :3]) and np.array_equal(qe.ext[ori_c, 3:], p.ext[ori_c, 3:])
    for g in range(p.n_group):
        const = [(int(p.group_const_mask[g]) >> j) & 1 == 1 for j in range(10)]
        assert np.array_equal(qe.intr[g][const], p.intr[g][const])


@pytest.mark.parametrize("name", sorted(vbo.SCENES))
def test_adjust_views_matches_oracle(oracle, name):
    p, kw = vbo.view_scene(name, n_cam=16, n_pt=600)
    views = list(range(1, p.n_cam, 1))                       # camera 0 stays out of the batch
    res_e, qe = run_engine(p, kw, views)
    res_o, qo = run_oracle(p, kw, views, oracle)
    compare(res_e, qe, res_o, qo, views, p)
    assert (res_e[3] > 0).sum() >= len(views) // 2


def test_degenerate_views(oracle):
    """No observations, no free coordinate, a failing functor: what the oracle returns, nothing touched."""
    p, kw = vbo.view_scene("radtan_per_camera_all", n_cam=8, n_pt=200)
    keep = p.obs_cam != 0
    p = _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const, p.obs_cam[keep],
                     p.obs_pt[keep], p.obs_xy[keep])
    p.ext_const[1] = _abi.EXT_ALL_CONST
    p.group_const_mask[p.cam_group[1]] = 0x3FF
    k = int(np.nonzero(p.obs_cam == 2)[0][0])
    p.pt[p.obs_pt[k]] = np.concatenate([p.ext[2, :3], [1.0]])
    views = list(range(p.n_cam))
    res_e, qe = run_engine(p, kw, views)
    res_o, qo = run_oracle(p, kw, views, oracle)
    compare(res_e, qe, res_o, qo, views, p)
    assert list(res_e[0][:3]) == [_abi.CONVERGENCE, _abi.CONVERGENCE, _abi.FAILURE] and list(res_e[3][:3]) == [0, 0, 0]
    assert np.array_equal(qe.ext[:3], p.ext[:3]) and np.array_equal(qe.intr[p.cam_group[:3]], p.intr[p.cam_group[:3]])


@pytest.mark.parametrize("n_obs", [1, 31, 32, 33, 255, 256, 257, 5000])
def test_cta_stride_edges(oracle, n_obs):
    """A view with exactly n_obs observations: the strided loops of the CTA's 128 threads and the warp staging at their edges."""
    p = synthetic.make_scene(n_cam=6, n_pt=n_obs, obs_per_pt=5, seed=40 + n_obs % 7, model=_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL,
                             shared_intrinsics=False, intrinsics_to_optimize=_abi.INTR_ALL, perturb=1.0)
    # camera 0 observes every point exactly once: drop its observations and add one per point, projected from the truth + noise
    rng = np.random.default_rng(n_obs)
    keep = p.obs_cam != 0
    truth_ext = p.ext[0].copy()
    pix, depth = synthetic.project(p.group_model[0], np.repeat(truth_ext[None], p.n_pt, 0), np.repeat(p.intr[p.cam_group[0]][None], p.n_pt, 0), p.pt)
    good = np.nonzero(depth > 0)[0]
    assert len(good) >= n_obs
    good = good[:n_obs]
    q = _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const,
                     np.concatenate([p.obs_cam[keep], np.zeros(n_obs, np.int32)]), np.concatenate([p.obs_pt[keep], good.astype(np.int32)]),
                     np.concatenate([p.obs_xy[keep], pix[good] + 0.3 * rng.normal(size=(n_obs, 2))]))
    q.ext[0, :3] += 0.02 * rng.normal(size=3); q.ext[0, 3:] += 0.002 * rng.normal(size=3)
    assert (q.obs_cam == 0).sum() == n_obs
    kw = dict(use_inner_iterations=0, linear_solver_type=_abi.DENSE_QR, max_num_iterations=50,
              intrinsics_to_optimize=_abi.INTR_FOCAL_LENGTH if n_obs < 8 else _abi.INTR_ALL)
    if n_obs < 8:
        q.group_const_mask[q.cam_group[0]] = 0x3FE
    views = [0]
    res_e, qe = run_engine(q, kw, views)
    res_o, qo = run_oracle(q, kw, views, oracle)
    compare(res_e, qe, res_o, qo, views, q)


def test_batch_larger_than_a_grid_wave(oracle):
    """More views than 132 SMs x resident CTAs; every view is independent, so each equals the same view adjusted alone."""
    p, kw = vbo.view_scene("pinhole_shared_none_huber", n_cam=900, n_pt=9000, obs_per_pt=4, seed=11)
    views = list(range(p.n_cam))
    res_e, qe = run_engine(p, kw, views)
    some = list(range(0, p.n_cam, 37))
    res_o, qo = run_oracle(p, kw, some, oracle)
    idx = np.array(some)
    st, ic, fc, it = res_e
    assert np.array_equal(st[idx], res_o[0]) and np.array_equal(it[idx], res_o[3])
    assert (rel_err(ic[idx], res_o[1]) <= 1e-11).all() and (rel_err(fc[idx], res_o[2]) <= 1e-7).all()
    assert np.abs(qe.ext[idx] - qo.ext[idx]).max() <= 1e-8 * np.abs(qo.ext).max()
    # the same views in a different batch composition give the same bits
    res_e2, qe2 = run_engine(p, kw, views[::-1])
    assert np.array_equal(qe2.ext, qe.ext) and np.array_equal(res_e2[2][::-1], fc)


def test_refusal_leaves_the_problem_untouched_and_solve_still_matches(oracle):
    p, kw = vbo.view_scene("pinhole_shared_default", n_cam=10, n_pt=400)
    q = p.copy()
    eng = engine.Engine()
    eng.upload(q, engine.default_options(**kw))
    for bad in ([0, 1], [3, 3], [p.n_cam], [-1]):
        with pytest.raises(engine.EngineError) as e:
            eng.adjust_views(engine.default_options(**kw), bad)
        assert e.value.code == _abi.ERR_INVALID_ARGUMENT
    eng.download(q)
    assert np.array_equal(q.ext, p.ext) and np.array_equal(q.intr, p.intr) and np.array_equal(q.pt, p.pt)
    eng.adjust_views(engine.default_options(**kw), [2])       # the camera-major index exists from here on
    eng.close()
    # a shared intrinsics group that is fully constant does not couple the views: one batch is accepted
    c = p.copy()
    c.group_const_mask[:] = 0x3FF
    ckw = dict(kw, intrinsics_to_optimize=_abi.INTR_NONE)
    eng = engine.Engine()
    eng.upload(c, engine.default_options(**ckw))
    st, _, _, _ = eng.adjust_views(engine.default_options(**ckw), list(range(c.n_cam)))
    eng.close()
    assert len(st) == c.n_cam and (st != _abi.FAILURE).all()
    # a full solve on a context that ran the views afterwards still equals the oracle
    skw = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, max_num_iterations=8)
    eng = engine.Engine()
    eng.upload(q, engine.default_options(**kw))
    eng.adjust_views(engine.default_options(**kw), [4])
    r = p.copy()
    sg = eng.solve(r, engine.default_options(**skw))
    eng.close()
    so = oracle.solve(p.copy(), oracle.default_options(**skw))
    assert sg.rc == 0 and abs(sg.initial_cost - so.initial_cost) <= 1e-12 * so.initial_cost
    assert np.all(np.abs(sg.costs - so.costs) <= 1e-8 * so.costs)
