"""Parity of the CUDA engine (through the C-ABI) against the CPU oracle and the committed golden
vectors.  Tolerances: fp64 everywhere; differences come only from summation order, FMA contraction
and the analytic-vs-autodiff evaluation of the same derivative, so
  * per-observation residual / Jacobian:            1e-12 relative (golden: torch.func.jacfwd)
  * cost, gradient, column norms, rhs, S*x:         1e-11 relative
  * SCHUR_JACOBI inverse blocks:                     1e-8  relative (inverse of blocks with cond ~1e4..1e6)
  * per-iteration cost trajectory, final cost:       1e-9 rel early, 1e-6 rel final (inexact PCG, eta = 0.1)
"""
import numpy as np
import pytest

from helpers import golden_problem, rel_err
from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu

ITER = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR)


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine()
    yield e
    e.close()


def _opts(mod, **kw):
    d = dict(ITER)
    d.update(kw)
    return mod.default_options(**d)


def test_jacobian_rows_match_golden(eng):
    """gradient = J^T r.  Two linearisations with r ~ e_0 and r ~ e_1 (measurement moved) give, per observation,
    G = Rm J with the 2x2 matrix Rm of the read-back residuals; J = Rm^-1 G is compared with the golden Jacobian."""
    prob, g = golden_problem()
    n = prob.n_obs
    pix = g["xy"] + g["r"]
    # a few random golden cases project near q_z = 0 (|pix| ~ 1e16): e_k cannot be represented next to pix there
    sane = np.abs(pix).max(axis=1) < 1e6
    assert sane.sum() >= 85
    G = np.zeros((n, 2, 20)); Rm = np.zeros((n, 2, 2))
    for row in (0, 1):
        p = prob.copy()
        p.group_const_mask[:] = 0  # every intrinsics column
        e = np.zeros(2); e[row] = 1.0
        p.obs_xy[:] = pix - e
        eng.upload(p, _opts(engine, intrinsics_to_optimize=_abi.INTR_ALL))
        ok, cost = eng.linearize()
        assert ok
        Rm[:, row, :] = eng.read(_abi.VEC_RESIDUALS).reshape(n, 2)
        G[:, row, :] = np.concatenate([eng.read(_abi.VEC_GRADIENT_CAM).reshape(n, 6), eng.read(_abi.VEC_GRADIENT_INTR).reshape(n, 10),
                                       eng.read(_abi.VEC_GRADIENT_PT).reshape(n, 4)], axis=1)
    assert np.abs(Rm[sane] - np.eye(2)).max() < 1e-9
    for i in np.nonzero(sane)[0]:
        J = np.linalg.solve(Rm[i], G[i])
        tol = 1e-12
        if str(g["tag"][i]) == "w_small_rodrigues":
            # theta ~ 2e-7: the jet evaluation of Rodrigues' formula cancels ((1-cos)/theta amplification),
            # the analytic form (2 sin^2(theta/2), series for (theta - sin)/theta^3) does not
            tol = 1e-7
        err = np.abs(J - g["J"][i]).max() / np.abs(g["J"][i]).max()
        assert err < tol, (i, str(g["tag"][i]), err)


def test_residuals_match_golden(eng):
    prob, g = golden_problem()
    eng.upload(prob, _opts(engine))
    ok, cost = eng.linearize()
    assert ok
    res = eng.read(_abi.VEC_RESIDUALS).reshape(-1, 2)
    scale = np.maximum(1.0, np.abs(g["r"]).max(axis=1))
    assert (np.abs(res - g["r"]).max(axis=1) / scale).max() < 1e-12
    assert abs(cost - 0.5 * (g["r"] ** 2).sum()) < 1e-11 * cost


ALL_LOSSES = [_abi.LOSS_TRIVIAL, _abi.LOSS_HUBER, _abi.LOSS_SOFTLONE, _abi.LOSS_CAUCHY, _abi.LOSS_ARCTAN, _abi.LOSS_TUKEY]

SCENES = {
    "pinhole_shared": dict(n_cam=12, n_pt=300, obs_per_pt=5, model=_abi.MODEL_PINHOLE, shared_intrinsics=True, seed=21),
    "radtan_per_camera": dict(n_cam=10, n_pt=400, obs_per_pt=6, model=_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, shared_intrinsics=False, seed=22),
    "radtan_all": dict(n_cam=10, n_pt=400, obs_per_pt=6, model=_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, shared_intrinsics=False, seed=23,
                       intrinsics_to_optimize=_abi.INTR_ALL),
    "pinhole_none": dict(n_cam=9, n_pt=200, obs_per_pt=4, model=_abi.MODEL_PINHOLE, shared_intrinsics=True, seed=24,
                         intrinsics_to_optimize=_abi.INTR_NONE),
    "pinhole_focal_pp": dict(n_cam=9, n_pt=200, obs_per_pt=4, model=_abi.MODEL_PINHOLE, shared_intrinsics=False, seed=25,
                             intrinsics_to_optimize=_abi.INTR_FOCAL_LENGTH | _abi.INTR_PRINCIPAL_POINTS),
    # tracks cut to 3..48 observations: 'long' tiles (tracks > 32 observations, per-point sums combined across warps in shared
    # memory) after the normal ones, with exactly-32 / 33-observation tracks at the boundary
    "long_short": dict(n_cam=120, n_pt=260, obs_per_pt=48, seed=41, track_lengths=(3, 7, 31, 32, 33, 48)),
}


def _width(loss, default):
    """Tukey's rho' is exactly 0 beyond its width: at the perturbed start (residuals of tens of pixels) a 2-pixel width would
    zero almost every Jacobian row and leave point blocks that consist of the LM diagonal only (cond ~1e10, rounding-level
    differences amplified to 1e-8).  A width that keeps the inliers inside exercises both of its branches instead."""
    return 80.0 if loss == _abi.LOSS_TUKEY else default


def _cut_tracks(p, lengths):
    """Every track keeps its first n observations, n drawn from `lengths` per point."""
    rng = np.random.default_rng(1)
    keep = np.ones(p.n_obs, bool)
    target = {q: int(rng.choice(lengths)) for q in range(p.n_pt)}
    seen = np.zeros(p.n_pt, int)
    for i in range(p.n_obs):
        q = int(p.obs_pt[i])
        seen[q] += 1
        keep[i] = seen[q] <= target[q]
    return _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const,
                        p.obs_cam[keep], p.obs_pt[keep], p.obs_xy[keep])


def _scene(name, constants=False):
    kw = dict(SCENES[name])
    lengths = kw.pop("track_lengths", None)
    p = synthetic.make_scene(**kw)
    if lengths is not None:
        p = _cut_tracks(p, lengths)
    if constants:
        p.ext_const[1] = _abi.EXT_ALL_CONST
        p.ext_const[2] = _abi.EXT_POSITION_CONST
        p.ext_const[3] = _abi.EXT_ORIENTATION_CONST
        p.pt_const[[5, 17]] = 1
    return p


@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("constants", [False, True])
@pytest.mark.parametrize("loss", ALL_LOSSES)
def test_stage_parity(eng, oracle, name, constants, loss):
    """Every stage of one LM iteration against the oracle, for all six LossFunctionType values (create_loss_function.cc:53-63)."""
    if constants and loss not in (_abi.LOSS_TRIVIAL, _abi.LOSS_HUBER, _abi.LOSS_TUKEY):
        pytest.skip("constant-block variants run with three of the six losses")
    p = _scene(name, constants)
    if loss != _abi.LOSS_TRIVIAL:
        p.obs_xy[::37] += 40.0  # outliers so that the robust branch is exercised
    kw = dict(loss_function_type=loss, robust_loss_width=_width(loss, 2.0))
    o = oracle.Oracle(p.copy(), _opts(oracle, **kw))
    eng.upload(p.copy(), _opts(engine, **kw))
    ok_o, cost_o = o.linearize()
    ok_g, cost_g = eng.linearize()
    assert ok_o and ok_g
    assert abs(cost_g - cost_o) <= 1e-12 * cost_o
    for which in (_abi.VEC_RESIDUALS, _abi.VEC_GRADIENT_CAM, _abi.VEC_GRADIENT_INTR, _abi.VEC_GRADIENT_PT,
                  _abi.VEC_COLNORM2_CAM, _abi.VEC_COLNORM2_INTR, _abi.VEC_COLNORM2_PT):
        a, b = eng.read(which), o.read(which)
        if np.abs(b).max() == 0:
            assert np.abs(a).max() == 0, which
        else:
            assert rel_err(a, b) < 1e-11, which
    radius = 1e4
    assert o.prepare_linear_system(radius) and eng.prepare_linear_system(radius)
    for which in (_abi.VEC_SCHUR_RHS_CAM, _abi.VEC_SCHUR_RHS_INTR):
        a, b = eng.read(which), o.read(which)
        if np.abs(b).max() > 0:
            assert rel_err(a, b) < 1e-10, which
    rng = np.random.default_rng(5)
    xc = rng.normal(size=p.n_cam * 6) * (o.read(_abi.VEC_COLNORM2_CAM) > 0)
    xi = rng.normal(size=p.n_group * 10) * (o.read(_abi.VEC_COLNORM2_INTR) > 0)
    # masked coordinates: the oracle's free mask = nonzero column norm here (generic geometry), except genuinely
    # constant coordinates which both sides must ignore
    yc_o, yi_o = o.schur_matvec(xc, xi)
    yc_g, yi_g = eng.schur_matvec(xc, xi)
    assert rel_err(yc_g, yc_o) < 1e-10
    if np.abs(yi_o).max() > 0:
        assert rel_err(yi_g, yi_o) < 1e-10
    Mc_o, Mc_g = o.read(_abi.VEC_PRECOND_CAM).reshape(-1, 36), eng.read(_abi.VEC_PRECOND_CAM).reshape(-1, 36)
    for c in range(p.n_cam):
        assert rel_err(Mc_g[c], Mc_o[c]) < 1e-8, c
    Mi_o, Mi_g = o.read(_abi.VEC_PRECOND_INTR).reshape(-1, 100), eng.read(_abi.VEC_PRECOND_INTR).reshape(-1, 100)
    for gi in range(p.n_group):
        assert rel_err(Mi_g[gi], Mi_o[gi]) < 1e-7, gi
    ok_o, it_o, mcc_o = o.solve_linear_system()
    ok_g, it_g, mcc_g = eng.solve_linear_system()
    assert ok_o and ok_g
    assert it_o == it_g, (it_o, it_g)
    assert abs(mcc_g - mcc_o) <= 1e-9 * abs(mcc_o)
    for which in (_abi.VEC_STEP_CAM, _abi.VEC_STEP_INTR, _abi.VEC_STEP_PT):
        a, b = eng.read(which), o.read(which)
        if np.abs(b).max() > 0:
            assert rel_err(a, b) < 1e-8, which
    ok_o, cand_o = o.evaluate_step()
    ok_g, cand_g = eng.evaluate_step()
    assert ok_o and ok_g and abs(cand_g - cand_o) <= 1e-9 * cand_o


@pytest.mark.parametrize("name", ["pinhole_shared", "radtan_per_camera", "pinhole_none"])
@pytest.mark.parametrize("loss", ALL_LOSSES)
def test_full_solve_parity(eng, oracle, name, loss):
    p0 = _scene(name, constants=(loss == _abi.LOSS_HUBER))
    kw = dict(loss_function_type=loss, robust_loss_width=_width(loss, 3.0), max_num_iterations=25)
    po, pg = p0.copy(), p0.copy()
    so = oracle.solve(po, _opts(oracle, **kw))
    sg = eng.solve(pg, _opts(engine, **kw))
    assert sg.rc == 0 and sg.success and so.success
    assert abs(sg.initial_cost - so.initial_cost) <= 1e-12 * so.initial_cost
    assert sg.num_iterations == so.num_iterations and sg.termination_type == so.termination_type, (sg.message, so.message)
    co, cg = so.costs, sg.costs
    n = len(co)
    assert np.all(np.abs(cg[:min(n, 10)] - co[:min(n, 10)]) <= 1e-9 * co[:min(n, 10)])
    assert np.all(np.abs(cg - co) <= 1e-6 * co)
    assert abs(sg.final_cost - so.final_cost) <= 1e-6 * so.final_cost
    assert [i["linear_solver_iterations"] for i in sg.iterations] == [i["linear_solver_iterations"] for i in so.iterations]
    # same trajectory => same parameters (no gauge alignment needed when the trajectories coincide)
    # (the re-descending losses ARCTAN / TUKEY flatten the cost around outliers: the same 1e-9 cost agreement leaves a looser hold
    # on the parameters along the weakly determined gauge directions -- 2.4e-6 seen with ARCTAN on pinhole_none)
    ptol = 1e-5 if loss in (_abi.LOSS_ARCTAN, _abi.LOSS_TUKEY) else 1e-6
    assert rel_err(pg.ext, po.ext) < ptol and rel_err(pg.pt, po.pt) < ptol and rel_err(pg.intr, po.intr) < ptol
    # constant blocks come back bit-identical (SubsetParameterization semantics)
    cm = p0.ext_const
    assert np.array_equal(pg.ext[cm == _abi.EXT_ALL_CONST], p0.ext[cm == _abi.EXT_ALL_CONST])
    assert np.array_equal(pg.ext[(cm & _abi.EXT_POSITION_CONST) != 0][:, :3], p0.ext[(cm & _abi.EXT_POSITION_CONST) != 0][:, :3])
    assert np.array_equal(pg.pt[p0.pt_const != 0], p0.pt[p0.pt_const != 0])


def test_config1_trajectory_matches_oracle(eng, oracle):
    """BASELINE.json configs[0]: 50 cameras / 5k points / 50k observations."""
    p0 = synthetic.make_config("c1_50cam")
    po, pg = p0.copy(), p0.copy()
    so = oracle.solve(po, _opts(oracle, max_num_iterations=30))
    sg = eng.solve(pg, _opts(engine, max_num_iterations=30))
    assert sg.rc == 0 and sg.success
    assert sg.num_iterations == so.num_iterations
    assert np.all(np.abs(sg.costs - so.costs) <= 1e-8 * so.costs)
    assert abs(sg.final_cost - so.final_cost) <= 1e-8 * so.final_cost
    # Camera::ProjectPoint consumers see the same per-track reprojection error (SURVEY 8c: <= 1e-8 px^2)
    ro, _, _ = oracle.residual_jacobian(po)
    rg, _, _ = oracle.residual_jacobian(pg)
    eo = np.bincount(po.obs_pt, weights=(ro ** 2).sum(1)) / np.bincount(po.obs_pt)
    eg = np.bincount(pg.obs_pt, weights=(rg ** 2).sum(1)) / np.bincount(pg.obs_pt)
    assert np.abs(eo - eg).max() < 1e-8


def test_edge_cases(eng, oracle):
    # empty problem
    p = _abi.Problem(np.zeros((0, 6)), [], [], [], np.zeros((0, 10)), [], np.zeros((0, 4)), [], [], [], np.zeros((0, 2)))
    s = eng.solve(p, _opts(engine))
    assert s.rc == 0 and s.success and s.initial_cost == 0.0
    # everything constant -> cost only
    q = _scene("pinhole_none")
    q.ext_const[:] = _abi.EXT_ALL_CONST
    q.pt_const[:] = 1
    q0 = q.copy()
    s = eng.solve(q, _opts(engine))
    so = oracle.solve(q0.copy(), _opts(oracle))
    assert s.rc == 0 and s.success and abs(s.initial_cost - so.initial_cost) <= 1e-12 * so.initial_cost
    assert s.final_cost == s.initial_cost and np.array_equal(q.pt, q0.pt) and np.array_equal(q.ext, q0.ext)
    # ragged track lengths, observation-less points and cameras, unsorted observation order
    r = _scene("pinhole_shared")
    keep = np.random.default_rng(3).uniform(size=r.n_obs) < 0.7
    keep[r.obs_pt == 7] = False
    keep[r.obs_cam == 4] = False
    perm = np.random.default_rng(4).permutation(int(keep.sum()))
    r = _abi.Problem(r.ext, r.ext_const, r.cam_group, r.group_model, r.intr, r.group_const_mask, r.pt, r.pt_const,
                     r.obs_cam[keep][perm], r.obs_pt[keep][perm], r.obs_xy[keep][perm])
    ro, rg = r.copy(), r.copy()
    so = oracle.solve(ro, _opts(oracle, max_num_iterations=15))
    sg = eng.solve(rg, _opts(engine, max_num_iterations=15))
    assert sg.rc == 0 and sg.num_iterations == so.num_iterations
    assert np.all(np.abs(sg.costs - so.costs) <= 1e-7 * so.costs)
    assert np.array_equal(rg.pt[7], r.pt[7]) and np.array_equal(rg.ext[4], r.ext[4])
    # point on top of a camera centre: evaluation fails at the initial point -> success = false
    f = _scene("pinhole_shared")
    f.pt[0, :3] = f.ext[f.obs_cam[f.obs_pt == 0][0], :3]
    f.pt[0, 3] = 1.0
    s = eng.solve(f, _opts(engine))
    assert s.rc == 0 and not s.success and s.termination_type == _abi.FAILURE
    # unsupported options fail loudly instead of silently doing something else
    s = eng.solve(_scene("pinhole_shared"), engine.default_options(linear_solver_type=6))  # CGNR
    assert s.rc == _abi.ERR_UNSUPPORTED and not s.success
    # a track longer than the engine limit is refused
    big = synthetic.make_scene(n_cam=600, n_pt=3, obs_per_pt=290, seed=1)
    s = eng.solve(big, _opts(engine))
    assert s.rc == _abi.ERR_UNSUPPORTED


def test_long_tracks_use_the_cta_level_path(eng, oracle):
    """Tracks with more than 32 observations live in 'long' tiles (per-point sums combined across warps in shared
    memory); mixed with short tracks and exactly-32 / 33-observation tracks at the boundary."""
    p = _scene("long_short")
    counts = np.bincount(p.obs_pt, minlength=p.n_pt)
    assert (counts > 32).sum() > 20 and (counts == 32).sum() > 5 and (counts < 32).sum() > 20
    po, pg = p.copy(), p.copy()
    so = oracle.solve(po, _opts(oracle, max_num_iterations=12))
    sg = eng.solve(pg, _opts(engine, max_num_iterations=12))
    assert sg.rc == 0 and sg.num_iterations == so.num_iterations
    assert np.all(np.abs(sg.costs - so.costs) <= 1e-8 * so.costs)
    assert rel_err(pg.pt, po.pt) < 1e-6 and rel_err(pg.ext, po.ext) < 1e-6


def test_schur_operator_properties_at_scale(eng):
    """Size-independent properties on a 200k-observation scene: S is symmetric positive definite and linear."""
    p = synthetic.make_scene(n_cam=200, n_pt=20_000, obs_per_pt=10, seed=9)
    eng.upload(p, _opts(engine))
    ok, cost = eng.linearize()
    assert ok and eng.prepare_linear_system(1e4)
    rng = np.random.default_rng(0)
    free_c = np.ones(p.n_cam * 6)
    free_i = np.zeros(p.n_group * 10); free_i[[0, 5, 6]] = 1
    a = (rng.normal(size=p.n_cam * 6) * free_c, rng.normal(size=p.n_group * 10) * free_i)
    b = (rng.normal(size=p.n_cam * 6) * free_c, rng.normal(size=p.n_group * 10) * free_i)
    Sa, Sb = eng.schur_matvec(*a), eng.schur_matvec(*b)
    dot = lambda u, v: float(u[0] @ v[0] + u[1] @ v[1])
    assert abs(dot(a, Sb) - dot(b, Sa)) <= 1e-9 * abs(dot(a, Sb))
    assert dot(a, Sa) > 0 and dot(b, Sb) > 0
    ab = (2.0 * a[0] - 3.0 * b[0], 2.0 * a[1] - 3.0 * b[1])
    Sab = eng.schur_matvec(*ab)
    assert rel_err(Sab[0], 2.0 * Sa[0] - 3.0 * Sb[0]) < 1e-10
    s = eng.minimize()
    assert s.success and s.final_cost < 0.01 * s.initial_cost
    costs = [i["cost"] for i in s.iterations if i["step_is_successful"]]
    assert all(y <= x for x, y in zip(costs, costs[1:]))


def test_not_positive_definite_system_is_an_invalid_step(oracle):
    """LM diagonal clamped to zero: the 4x4 block of a homogeneous point is singular, the Cholesky factorisation fails and every step
    is invalid (trust_region_minimizer.cc HandleInvalidStep) until max_num_consecutive_invalid_steps ends the solve with FAILURE.  The
    engine learns about the failed factorisation only together with the PCG's termination state (deferred flag, stage_pcg): the
    iterations that ran on the unusable system must leave no trace -- same log as the oracle, parameters untouched."""
    p = synthetic.make_scene(n_cam=12, n_pt=300, obs_per_pt=10, seed=4)
    kw = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, min_lm_diagonal=0.0, max_lm_diagonal=0.0, max_num_iterations=10)
    po, pg = p.copy(), p.copy()
    so = oracle.solve(po, oracle.default_options(**kw))
    eng = engine.Engine()
    sg = eng.solve(pg, engine.default_options(**kw))
    eng.close()
    assert so.termination_type == _abi.FAILURE and sg.termination_type == _abi.FAILURE
    assert sg.num_iterations == so.num_iterations and np.allclose(sg.costs, so.costs, rtol=1e-12)
    assert all(it["linear_solver_iterations"] == 0 and not it["step_is_valid"] for it in sg.iterations[1:])
    assert np.array_equal(pg.ext, p.ext) and np.array_equal(pg.pt, p.pt) and np.array_equal(pg.intr, p.intr)
