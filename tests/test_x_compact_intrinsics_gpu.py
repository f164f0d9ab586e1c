"""The compact layout of the stored linearisation: with one shared intrinsics group, the TRIVIAL loss and NI >= 2 free intrinsics
columns, J stores the normalised image point (u, v) in place of J_i, and every pass over J rebuilds J_i from it.  The same scene is
uploaded twice: with the TRIVIAL loss (compact layout) and with a HUBER loss whose width no residual reaches (the same arithmetic:
rho = s, rho' = 1, rho'' = 0, the corrector is the identity; full layout).  The rebuilt J_i must equal the stored one bit for bit,
on the normal tiles (k_linearize_stream) and the long tiles (k_linearize), and the rows both layouts share must be identical."""
import numpy as np
import pytest

from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu

PINHOLE, RADTAN = _abi.MODEL_PINHOLE, _abi.MODEL_PINHOLE_RADIAL_TANGENTIAL
DEFAULT = _abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION
# name: (model, intrinsics_to_optimize, NI)
CASES = {
    "pinhole_none": (PINHOLE, _abi.INTR_NONE, 0),
    "pinhole_default": (PINHOLE, DEFAULT, 3),
    "radtan_default": (RADTAN, DEFAULT, 4),
    "pinhole_all": (PINHOLE, _abi.INTR_ALL, 7),
    "radtan_all": (RADTAN, _abi.INTR_ALL, 10),
}
TRACKS = (3, 7, 31, 32, 33, 48)


def _scene(model, intr, seed):
    """normal and long tiles (tracks of 3..48 observations), constant blocks (zeroed rows) and outliers"""
    p = synthetic.make_scene(n_cam=120, n_pt=260, obs_per_pt=48, seed=seed, model=model, shared_intrinsics=True,
                             intrinsics_to_optimize=intr)
    rng = np.random.default_rng(seed)
    target = rng.choice(TRACKS, size=p.n_pt)
    seen = np.zeros(p.n_pt, int)
    keep = np.ones(p.n_obs, bool)
    for i in range(p.n_obs):
        q = int(p.obs_pt[i])
        seen[q] += 1
        keep[i] = seen[q] <= target[q]
    p = _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const,
                     p.obs_cam[keep], p.obs_pt[keep], p.obs_xy[keep])
    p.ext_const[1] = _abi.EXT_ALL_CONST
    p.ext_const[2] = _abi.EXT_POSITION_CONST
    p.pt_const[[5, 17, 40]] = 1
    p.obs_xy[::37] += 40.0
    return p


def _options(intr, loss):
    wide = dict(loss_function_type=_abi.LOSS_HUBER, robust_loss_width=1e30) if loss == "huber_wide" else {}
    return engine.default_options(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, intrinsics_to_optimize=intr,
                                  max_num_iterations=8, **wide)


def _linearise(p, opts, tile_kernel):
    eng = engine.Engine()
    try:
        eng.upload(p, opts)
        lin = eng.linearize_raw(tile_kernel=tile_kernel)
        lin["Ji"] = eng.intr_cols_raw()
        lin["nj"] = eng.profile()["doubles_per_obs"]
    finally:
        eng.close()
    return lin


@pytest.mark.parametrize("tile_kernel", [False, True], ids=["streaming", "tile"])
@pytest.mark.parametrize("name", list(CASES))
def test_rebuilt_intrinsics_columns_equal_the_stored_ones(request, name, tile_kernel):
    if request.config.getoption("--mock-engine"):
        pytest.skip("raw device buffers: the real engine or its emulation build only")
    model, intr, ni = CASES[name]
    p = _scene(model, intr, seed=71 + ni)
    assert engine.debug_pack(p)["NI"] == ni
    flags = engine.debug_pack(p)["tile_flags"]
    assert (flags & 1).any() and not (flags & 1).all(), "the scene must have normal and long tiles"
    a = _linearise(p, _options(intr, "trivial"), tile_kernel)
    b = _linearise(p, _options(intr, "huber_wide"), tile_kernel)
    assert b["nj"] == 14 + 2 * ni, "a robust loss keeps the full layout"
    assert a["nj"] == (16 if ni >= 2 else 14 + 2 * ni)
    assert a["failed"] == 0.0 and b["failed"] == 0.0
    assert a["J"].shape[1] == a["nj"] and b["J"].shape[1] == b["nj"]
    assert np.array_equal(a["J"][:, :14], b["J"][:, :14])
    assert np.array_equal(a["res"], b["res"])
    assert abs(a["cost"] - b["cost"]) <= 1e-12 * b["cost"]  # sums of fp64 atomics
    # J_i as every pass over J sees it: rebuilt from (u, v) in the compact layout, bit for bit the rows the full layout stores
    assert a["Ji"].shape == b["Ji"].shape == (len(b["J"]), 2 * ni, 32)
    assert np.array_equal(b["Ji"], b["J"][:, 14:])
    assert np.array_equal(a["Ji"], b["J"][:, 14:])
    if ni >= 2:
        assert np.abs(a["Ji"]).max() > 0.0
        # zeroed rows (padding, constant blocks) are marked by a NaN u; every other slot stores its normalised image point
        zeroed = np.all(b["J"][:, :14] == 0.0, axis=1)
        assert zeroed.any() and not zeroed.all()
        assert np.isnan(a["J"][:, 14][zeroed]).all() and np.isfinite(a["J"][:, 14:16].transpose(0, 2, 1)[~zeroed]).all()


@pytest.mark.parametrize("name", ["pinhole_default", "radtan_all"])
def test_solve_on_the_compact_layout_follows_the_full_layout(request, name):
    """the whole LM solve: equal up to the order of the fp64 atomics"""
    if request.config.getoption("--mock-engine"):
        pytest.skip("compares two layouts of the real engine")
    model, intr, ni = CASES[name]
    p = _scene(model, intr, seed=91 + ni)
    out = {}
    for loss in ("trivial", "huber_wide"):
        eng = engine.Engine()
        try:
            out[loss] = eng.solve(p.copy(), _options(intr, loss))
        finally:
            eng.close()
    a, b = out["trivial"], out["huber_wide"]
    assert a.rc == 0 and b.rc == 0 and a.success and b.success
    assert abs(a.initial_cost - b.initial_cost) <= 1e-13 * b.initial_cost
    assert len(a.costs) == len(b.costs)
    assert np.all(np.abs(a.costs - b.costs) <= 1e-9 * b.costs), (a.costs, b.costs)
