"""N3 on the GPU, through the C-ABI: tba_estimate_tracks (batched TrackEstimator::EstimateTrack) and tba_adjust_tracks
(batched BundleAdjustTrack) on the device-resident problem, against the oracle's per-track restatement.  The same device
bodies are checked on the host by tests/test_track_estimator.py and tests/test_point_lm.py; this file adds the kernels,
the upload / download glue and the packed <-> caller scatter.  Never executed on hardware in round 1 (GPU budget spent)."""
import numpy as np
import pytest

from helpers import fountain_problem, long_track_scene
from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu
KW = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR)


def euclid(x):
    return x[:, :3] / x[:, 3:4]


@pytest.mark.parametrize("model", [_abi.MODEL_PINHOLE, _abi.MODEL_PINHOLE_RADIAL_TANGENTIAL])
@pytest.mark.parametrize("ba", [True, False])
def test_estimate_tracks_matches_oracle(oracle, model, ba):
    p = synthetic.make_scene(n_cam=60, n_pt=5000, obs_per_pt=5, seed=33, model=model, noise_px=0.5, perturb=0.0)
    rng = np.random.default_rng(2)
    p.obs_xy[rng.choice(p.n_obs, 200, replace=False)] += 300.0           # tracks that must fail the reprojection test
    p.pt[:] = rng.normal(size=p.pt.shape)                                  # incoming value is ignored
    p.pt_const[::97] = 1                                                   # "already estimated": skipped, bit-identical
    st = _estimate_and_compare(oracle, p, ba, const=slice(None, None, 97))
    assert (st == 0).sum() > 4000 and (st == 4).sum() >= 100


@pytest.mark.parametrize("ba", [True, False])
def test_estimate_tracks_on_long_tracks(oracle, ba):
    """Tracks of 33..256 observations (helpers.long_track_scene): k_estimate_tracks walks each one over the warp slices of a
    long tile."""
    p = long_track_scene(seed=33, filler=40, noise_px=0.5, perturb=0.0)
    rng = np.random.default_rng(2)
    for q in rng.choice(p.n_pt, 8, replace=False):
        p.obs_xy[np.nonzero(p.obs_pt == q)[0][:3]] += 300.0              # tracks that must fail the reprojection test
    p.pt[:] = rng.normal(size=p.pt.shape)
    p.pt_const[::7] = 1
    st = _estimate_and_compare(oracle, p, ba, const=slice(None, None, 7))
    assert (st == 0).sum() >= 40 and (st == 4).sum() >= 5


def _estimate_and_compare(oracle, p, ba, const):
    before = p.pt.copy()
    q = p.copy()
    st_o, counts_o = oracle.estimate_tracks(q, oracle.default_options(**KW), bundle_adjustment=ba)
    eng = engine.Engine()
    eng.upload(p, engine.default_options(**KW))
    st, counts = eng.estimate_tracks(engine.default_options(**KW), 5.0, 3.0, ba)
    eng.download(p)
    eng.close()
    assert np.array_equal(st, st_o) and np.array_equal(counts, counts_o)
    assert (st[const] == 255).all() and np.array_equal(p.pt[const], before[const])
    ok = st == 0
    tol = 1e-6 if ba else 1e-10
    assert np.abs(euclid(p.pt[ok]) - euclid(q.pt[ok])).max() <= tol * np.abs(euclid(q.pt[ok])).max()
    return st


def test_adjust_tracks_matches_oracle(oracle):
    p = synthetic.make_scene(n_cam=40, n_pt=3000, obs_per_pt=6, seed=19)   # perturbed points, cameras held where they are
    p.pt_const[::50] = 1
    _adjust_and_compare(oracle, p, const=slice(None, None, 50))


def test_adjust_tracks_on_long_tracks(oracle):
    """BundleAdjustTrack over tracks of 33..256 observations (helpers.long_track_scene), with outliers under HUBER."""
    p = long_track_scene(seed=19, filler=40)
    p.pt_const[::9] = 1
    p.obs_xy[::23] += 30.0
    _adjust_and_compare(oracle, p, const=slice(None, None, 9))


def _adjust_and_compare(oracle, p, const):
    q = p.copy()
    opts = dict(KW, loss_function_type=_abi.LOSS_HUBER, robust_loss_width=3.0)
    st_o, ic_o, fc_o, failed_o = oracle.adjust_tracks(q, oracle.default_options(**opts))
    eng = engine.Engine()
    eng.upload(p, engine.default_options(**opts))
    st, ic, fc, failed = eng.adjust_tracks(engine.default_options(**opts))
    eng.download(p)
    eng.close()
    assert np.array_equal(st == 255, st_o == 255) and (st[const] == 255).all()
    live = st != 255
    assert np.allclose(ic[live], ic_o[live], rtol=1e-11)
    # a track that has not converged after max_num_iterations (one of 2940 in the oracle run) sits in a flat valley where
    # FMA-level differences decide the last steps: terminations must agree on all but a handful, values on the converged ones
    assert (st != st_o).sum() <= 3 and abs(failed - failed_o) <= 3
    conv = live & (st == _abi.CONVERGENCE) & (st_o == _abi.CONVERGENCE)
    assert conv.sum() >= live.sum() - 6
    assert np.allclose(fc[conv], fc_o[conv], rtol=1e-7, atol=1e-12)
    assert np.abs(euclid(p.pt[conv]) - euclid(q.pt[conv])).max() <= 1e-6 * np.abs(euclid(q.pt[conv])).max()
    assert np.array_equal(p.ext, q.ext) and np.array_equal(p.intr, q.intr)   # cameras untouched


def test_estimate_tracks_on_the_reference_fountain(oracle):
    p, g = fountain_problem()
    ref = p.pt.copy()
    p.pt[:] = 0.0
    eng = engine.Engine()
    eng.upload(p, engine.default_options(**KW))
    st, counts = eng.estimate_tracks(engine.default_options(**KW))
    eng.download(p)
    # the refined tracks then pass the post-BA filter on the same context
    fst, mean, nb, ni = eng.filter_tracks(5.0, 3.0)
    eng.close()
    ok = st == 0
    assert ok.mean() > 0.995 and counts[0] == ok.sum()
    scale = np.linalg.norm(euclid(ref) - euclid(ref).mean(0), axis=1).mean()
    err = np.linalg.norm(euclid(p.pt[ok]) - euclid(ref[ok]), axis=1)
    assert np.median(err) < 2e-3 * scale
    assert (fst[ok] == 0).mean() > 0.999
