"""N1 on the GPU: tba_filter_tracks evaluated on the device-resident problem right after a solve, against the oracle's
restatement on the parameters the solve returned.  First executed by the round-end driver (DESIGN.md 7.4)."""
import numpy as np
import pytest

from helpers import fountain_problem, long_track_scene
from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu
KW = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, max_num_iterations=8)


def _check(eng, oracle, p, thresholds):
    s = eng.solve(p, engine.default_options(**KW))   # p now holds the refined parameters; the device copy is resident
    assert s.rc == 0
    statuses = []
    for max_err, angle in thresholds:
        st, mean, nb, ni = eng.filter_tracks(max_err, angle)
        st_o, mean_o, removed = oracle.filter_tracks(p, max_err, angle)
        ok = np.isfinite(mean_o)
        assert np.allclose(mean[ok], mean_o[ok], rtol=1e-9, atol=1e-12)
        # a track whose statistic sits within rounding of a threshold may fall on either side
        borderline = ok & (np.abs(mean_o - max_err ** 2) <= 1e-9 * max_err ** 2)
        assert np.array_equal(st[~borderline], st_o[~borderline])
        assert abs((nb + ni) - removed) <= int(borderline.sum())
        statuses.append(st_o)
    return np.concatenate(statuses)


def test_filter_matches_oracle_on_synthetic_with_outliers(oracle):
    p = synthetic.make_scene(n_cam=40, n_pt=3000, obs_per_pt=7, seed=14)
    rng = np.random.default_rng(3)
    p.obs_xy[rng.choice(p.n_obs, 150, replace=False)] += 30.0
    p.pt_const[:] = 0
    eng = engine.Engine()
    _check(eng, oracle, p, [(5.0, 3.0), (1.0, 1.0), (0.6, 20.0)])
    eng.close()


def test_filter_matches_oracle_on_long_tracks(oracle):
    """Tracks of 33..256 observations (helpers.long_track_scene): k_filter_tracks walks each one over the warp slices of a long
    tile, from mid-warp starts and across padding.  The thresholds give all three outcomes."""
    p = long_track_scene(seed=14, filler=40)
    rng = np.random.default_rng(3)
    p.obs_xy[rng.choice(p.n_obs, 40, replace=False)] += 30.0
    eng = engine.Engine()
    st = _check(eng, oracle, p, [(5.0, 3.0), (3.0, 1.0), (5.0, 60.0)])
    eng.close()
    assert set(np.unique(st).tolist()) == {0, 1, 2}


def test_filter_on_the_reference_fountain_reconstruction(oracle):
    p, g = fountain_problem()
    eng = engine.Engine()
    _check(eng, oracle, p, [(5.0, 3.0), (1.0, 3.0)])
    st, mean, nb, ni = eng.filter_tracks(5.0, 3.0)
    assert nb + ni <= 10
    eng.close()
