"""TEST INFRASTRUCTURE: BundleAdjustView (bundle_adjustment.cc:83-93) restated serially for the tests of tba_adjust_views.

Per view: one reprojection residual per observation of the camera, every point constant, the camera's extrinsics and its
intrinsics group free where ext_const / group_const_mask leave them free, DENSE_QR, no inner iterations -- Ceres' trust-region
loop (the control flow of oracle_solve) on that one dense block.  Residuals and Jacobians come from the oracle's jets
(oracle_py.residual_jacobian), the robust loss from the oracle's loss (oracle_py.loss), the linear algebra from numpy: nothing
here shares code with the engine.  test_view_ba.py checks this restatement against oracle_py.solve on the single-view
sub-problems (single_view_problem)."""
import numpy as np

from oracle import oracle_py
from theiasfm_b200 import _abi

DBL_MAX = np.finfo(np.float64).max


def free_mask(problem, cam):
    """[16] bool: which of [C (3) | w (3) | intrinsics (10)] the view optimises."""
    g = int(problem.cam_group[cam]); K = _abi.MODEL_NUM_PARAMS[int(problem.group_model[g])]
    ec = int(problem.ext_const[cam]); gm = int(problem.group_const_mask[g])
    fm = np.zeros(16, bool)
    fm[:3] = not ec & _abi.EXT_POSITION_CONST
    fm[3:6] = not ec & _abi.EXT_ORIENTATION_CONST
    fm[6:6 + K] = [not (gm >> j) & 1 for j in range(K)]
    return fm


def single_view_problem(problem, cam):
    """The problem BundleAdjustView(cam) hands to Ceres: that camera, its intrinsics group, its observations, their points
    (constant).  Returns (sub-problem, observed caller point indices)."""
    sel = np.nonzero(problem.obs_cam == cam)[0]
    pts, op = np.unique(problem.obs_pt[sel], return_inverse=True)
    g = int(problem.cam_group[cam])
    sub = _abi.Problem(problem.ext[cam:cam + 1].copy(), problem.ext_const[cam:cam + 1], np.zeros(1, np.int32), problem.group_model[g:g + 1],
                       problem.intr[g:g + 1].copy(), problem.group_const_mask[g:g + 1], problem.pt[pts].copy(), np.ones(len(pts), np.uint8),
                       np.zeros(len(sel), np.int32), op.astype(np.int32), problem.obs_xy[sel])
    return sub, pts


def _evaluate(sub, fm, options, derivs):
    """Cost (and H, g of the masked, robustified Jacobian) of the sub-problem at its current ext / intr; None on a failed functor."""
    r, J, ok = oracle_py.residual_jacobian(sub)
    if not ok.all():
        return None
    s = (r * r).sum(axis=1)
    if options.loss_function_type == _abi.LOSS_TRIVIAL:
        rho = np.stack([s, np.ones_like(s), np.zeros_like(s)], axis=1)
    else:
        rho = np.array([oracle_py.loss(options.loss_function_type, options.robust_loss_width, si) for si in s]).reshape(-1, 3)
    cost = 0.5 * rho[:, 0].sum()
    if not derivs:
        return cost
    Jc = J[:, :, :16] * fm[None, None, :]
    # Corrector (corrector.cc)
    sq1 = np.sqrt(rho[:, 1])
    plain = (s == 0.0) | (rho[:, 2] <= 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        alpha = np.where(plain, 0.0, 1.0 - np.sqrt(1.0 + 2.0 * s * rho[:, 2] / rho[:, 1]))
        rscale = np.where(plain, sq1, sq1 / (1.0 - alpha))
        asn = np.where(plain, 0.0, alpha / s)
    rtj = np.einsum("ka,kaj->kj", r, Jc)
    Jr = sq1[:, None, None] * (Jc - asn[:, None, None] * r[:, :, None] * rtj[:, None, :])
    rr = r * rscale[:, None]
    return cost, Jr, rr


def _view_lm(sub, fm, options):
    """oracle_solve's trust-region loop with the exact solver on one block.  Returns (termination, initial, final, iterations)."""
    o = options
    K = _abi.MODEL_NUM_PARAMS[int(sub.group_model[0])]
    blk = np.zeros(16, bool)
    blk[:6] = fm[:6].any()
    blk[6:6 + K] = fm[6:].any()

    def get():
        return np.concatenate([sub.ext[0], sub.intr[0]])

    def put(u):
        sub.ext[0] = u[:6]; sub.intr[0] = u[6:]

    x = get()
    e = _evaluate(sub, fm, o, True)
    if e is None:
        return _abi.FAILURE, -1.0, -1.0, 0
    cost, Jr, rr = e
    initial = cost
    g = np.einsum("kaj,ka->j", Jr, rr)
    cn = np.einsum("kaj,kaj->j", Jr, Jr)
    scale = 1.0 / (1.0 + np.sqrt(cn)) if o.jacobi_scaling else np.ones(16)
    gmax = np.abs(g).max()
    xnorm = np.sqrt((x[blk] ** 2).sum())
    radius, decrease = o.initial_trust_region_radius, 2.0
    invalid, rows, successful = 0, 0, True
    term = _abi.NO_CONVERGENCE
    while True:
        rows += 1                                              # iteration rows-1 is listed
        it = rows - 1
        if it >= o.max_num_iterations:
            term = _abi.NO_CONVERGENCE; break
        if successful and gmax <= o.gradient_tolerance:
            term = _abi.CONVERGENCE; break
        if radius <= o.min_trust_region_radius:
            term = _abi.CONVERGENCE; break
        Js = Jr * scale[None, None, :]
        diag = np.clip(np.einsum("kaj,kaj->j", Js, Js), o.min_lm_diagonal, o.max_lm_diagonal)
        D = np.where(fm, np.sqrt(diag / radius), 0.0)
        f = np.nonzero(fm)[0]
        xs = np.zeros(16)
        valid = True
        if len(f):
            S = np.einsum("kai,kaj->ij", Js[:, :, f], Js[:, :, f]) + np.diag(D[f] * D[f])
            b = np.einsum("kaj,ka->j", Js[:, :, f], rr)
            try:
                Lc = np.linalg.cholesky(S)
                xs[f] = np.linalg.solve(Lc.T, np.linalg.solve(Lc, b))
            except np.linalg.LinAlgError:
                valid = False
        mcc = 0.0
        if valid:
            m = -np.einsum("kaj,j->ka", Js, xs)
            mcc = -(m * (rr + m / 2.0)).sum()
            delta = -xs * scale
            valid = bool(np.isfinite(delta).all()) and mcc > 0.0
        if not valid:
            invalid += 1
            if invalid >= o.max_num_consecutive_invalid_steps:
                term = _abi.FAILURE; break
            radius /= decrease; decrease *= 2.0; successful = False
            continue
        invalid = 0
        cand = x.copy(); cand[fm] += delta[fm]
        put(cand)
        cc = _evaluate(sub, fm, o, False)
        cc = DBL_MAX if cc is None else cc
        step_norm = np.sqrt(((x - cand)[blk] ** 2).sum())
        if step_norm <= o.parameter_tolerance * (xnorm + o.parameter_tolerance):
            put(x); term = _abi.CONVERGENCE; break
        change = cost - cc
        if abs(change) <= o.function_tolerance * cost:
            put(x); term = _abi.CONVERGENCE; break
        rel = change / mcc
        if rel > o.min_relative_decrease:
            x = cand
            xnorm = np.sqrt((x[blk] ** 2).sum())
            e = _evaluate(sub, fm, o, True)
            if e is None:
                term = _abi.FAILURE; break
            cost, Jr, rr = e
            g = np.einsum("kaj,ka->j", Jr, rr)
            gmax = np.abs(g).max()
            radius = min(o.max_trust_region_radius, radius / max(1.0 / 3.0, 1.0 - (2.0 * rel - 1.0) ** 3))
            decrease, successful = 2.0, True
        else:
            put(x)
            radius /= decrease; decrease *= 2.0; successful = False
    put(x)
    return term, initial, cost, rows - 1


def check_views(problem, views):
    """The refusals of tba_adjust_views, as an error code (_abi.OK when the batch is valid)."""
    views = [int(v) for v in views]
    if any(v < 0 or v >= problem.n_cam for v in views) or len(set(views)) != len(views):
        return _abi.ERR_INVALID_ARGUMENT
    groups = [int(problem.cam_group[v]) for v in views if free_mask(problem, v)[6:].any()]
    return _abi.OK if len(set(groups)) == len(groups) else _abi.ERR_INVALID_ARGUMENT


def adjust_views(problem, options, views):
    """Batched BundleAdjustView, one view after another; updates problem.ext / problem.intr in place.
    Returns (status [n] uint8, initial_cost, final_cost, iterations [n] int32).  Raises ValueError on a refused batch."""
    rc = check_views(problem, views)
    if rc != _abi.OK:
        raise ValueError("tba_adjust_views refuses this batch (%d)" % rc)
    n = len(views)
    st = np.zeros(n, np.uint8); ic = np.zeros(n); fc = np.zeros(n); it = np.zeros(n, np.int32)
    for i, cam in enumerate(views):
        cam = int(cam)
        sub, _ = single_view_problem(problem, cam)
        st[i], ic[i], fc[i], it[i] = _view_lm(sub, free_mask(problem, cam), options)
        problem.ext[cam] = sub.ext[0]
        problem.intr[int(problem.cam_group[cam])] = sub.intr[0]
    return st, ic, fc, it


def extend_mock_engine():
    """Under `pytest --mock-engine`, give the stand-in engine an adjust_views answered by this restatement."""
    import sys
    mock = sys.modules.get("mock_engine_py")
    if mock is None or hasattr(mock.MockEngine, "adjust_views"):
        return

    def mock_adjust_views(self, options, views):
        from theiasfm_b200 import engine
        if check_views(self._w, views) != _abi.OK:
            raise engine.EngineError(_abi.ERR_INVALID_ARGUMENT, "refused batch")
        return adjust_views(self._w, options, views)

    mock.MockEngine.adjust_views = mock_adjust_views


# ------------------------------------------------------------------------------------------------ scenes of the view tests
# name -> (camera model, shared intrinsics group, intrinsics_to_optimize, loss, constant orientation, constant position)
SCENES = {
    "pinhole_shared_default": (_abi.MODEL_PINHOLE, True, _abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION, _abi.LOSS_TRIVIAL, 0, 0),
    "pinhole_shared_none_huber": (_abi.MODEL_PINHOLE, True, _abi.INTR_NONE, _abi.LOSS_HUBER, 0, 0),
    "radtan_per_camera_all": (_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, False, _abi.INTR_ALL, _abi.LOSS_TRIVIAL, 0, 0),
    "radtan_cauchy_const_orientation": (_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, False, _abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION,
                                        _abi.LOSS_CAUCHY, 1, 0),
    "pinhole_const_position_all": (_abi.MODEL_PINHOLE, False, _abi.INTR_ALL, _abi.LOSS_TRIVIAL, 0, 1),
    "fisheye_per_camera_default": (_abi.MODEL_FISHEYE, False, _abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION, _abi.LOSS_TRIVIAL, 0, 0),
    "fov_per_camera_all": (_abi.MODEL_FOV, False, _abi.INTR_ALL, _abi.LOSS_HUBER, 0, 0),
    "division_per_camera_default": (_abi.MODEL_DIVISION_UNDISTORTION, False, _abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION,
                                    _abi.LOSS_TRIVIAL, 0, 0),
}


def view_scene(name, n_cam=12, n_pt=300, obs_per_pt=4, seed=5):
    """(problem, options kwargs) of a SCENES entry: cameras perturbed, points near the truth; ext_const / group_const_mask filled
    from the options the way the adapter fills them."""
    from theiasfm_b200 import synthetic
    model, shared, intr_opt, loss, c_orient, c_pos = SCENES[name]
    p = synthetic.make_scene(n_cam=n_cam, n_pt=n_pt, obs_per_pt=obs_per_pt, model=model, shared_intrinsics=shared, seed=seed,
                             intrinsics_to_optimize=intr_opt, perturb=1.0)
    p.ext_const[:] = (_abi.EXT_ORIENTATION_CONST if c_orient else 0) | (_abi.EXT_POSITION_CONST if c_pos else 0)
    if loss != _abi.LOSS_TRIVIAL:
        rng = np.random.default_rng(seed)
        p.obs_xy[rng.choice(p.n_obs, max(1, p.n_obs // 50), replace=False)] += 25.0   # outliers for the robust loss
    kw = dict(loss_function_type=loss, robust_loss_width=2.0, constant_camera_orientation=c_orient, constant_camera_position=c_pos,
              intrinsics_to_optimize=intr_opt, use_inner_iterations=0, linear_solver_type=_abi.DENSE_QR, max_num_iterations=50)
    return p, kw


def batches(problem, views):
    """Split views, in order, into consecutive batches that tba_adjust_views accepts (a free intrinsics group at most once per batch):
    adjusting them batch after batch is the sequential BundleAdjustView of the list."""
    out, cur, used = [], [], set()
    for v in views:
        g = int(problem.cam_group[v])
        if free_mask(problem, v)[6:].any() and g in used:
            out.append(cur); cur, used = [], set()
        cur.append(int(v))
        if free_mask(problem, v)[6:].any():
            used.add(g)
    if cur:
        out.append(cur)
    return out
