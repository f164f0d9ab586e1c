"""Stage parity on long tiles: tracks of 33 to 256 observations.

A track of more than 32 observations goes to a long tile, the only layout where a point straddles warp slices and where several
points share a tile at arbitrary offsets.  Long tiles take their own kernels: k_linearize (per-point sums combined in shared
memory), k_schur MODE 0 / 1 / 2 (one CTA per tile), and the SCHUR_JACOBI blocks k_precond_ext and k_precond_intr, the latter
driven by the pack's per-tile (point, intrinsics group) runs (slot_run, tile_nruns).  Each scene is laid out track by track
(helpers.long_track_scene) and asserts from the host pack the layouts it exists for: a tile holding one 256-observation point, one
holding a 255-observation point and a padding slot, points starting mid-warp over three or more warp slices, points ending on a
warp boundary and one slot past it, a tile of seven points, 256 runs in one tile (per-camera intrinsics), and problems without
normal tiles (the long kernels then start at tile 0).  Each scene walks one LM iteration against the oracle block by block
(helpers.block_err), as test_x_stream_ranges_gpu does for the normal tiles."""
import numpy as np
import pytest

from helpers import block_err, long_track_scene, packed_extents
from theiasfm_b200 import _abi, engine

pytestmark = pytest.mark.gpu

PINHOLE, RADTAN, FISHEYE = _abi.MODEL_PINHOLE, _abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, _abi.MODEL_FISHEYE
FOCAL_RADIAL = _abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION


def _constants_and_outliers(p):
    p.ext_const[1] = _abi.EXT_ALL_CONST
    p.ext_const[2] = _abi.EXT_POSITION_CONST
    p.ext_const[3] = _abi.EXT_ORIENTATION_CONST
    p.pt_const[[1, 3, 12, 25]] = 1  # the 255-observation point, the mid-warp one, the one ending at slot 65, a filler track
    p.obs_xy[::37] += 40.0          # outliers for the robust branch


# scene: make_scene arguments; filler: more long tracks of 33..256 after helpers.LONG_LAYOUT; short: tracks of 2..32 (normal tiles);
# imask: the intrinsics column set the engine must dispatch
SCENES = {
    # per-camera intrinsics: one 256-observation point over 256 groups = 256 runs in its tile (k_precond_intr, multi-group)
    "radtan_per_camera": dict(scene=dict(model=RADTAN, shared_intrinsics=False, seed=61), filler=24, short=0, imask=0x0E1),
    # one shared group: k_precond_intr's single_group replica path
    "pinhole_shared_all": dict(scene=dict(model=PINHOLE, seed=62, intrinsics_to_optimize=_abi.INTR_ALL), filler=24, short=400,
                               imask=0x07F),
    "pinhole_none": dict(scene=dict(model=PINHOLE, seed=63, intrinsics_to_optimize=_abi.INTR_NONE), filler=24, short=400, imask=0x000),
    # EXT camera model: every tile through k_linearize<0x3FF, true>, whose per-lane RED branch is not staged
    "fisheye_per_camera": dict(scene=dict(model=FISHEYE, shared_intrinsics=False, seed=64), filler=16, short=300, imask=0x3FF,
                               ext=True),
    # no SCHUR_JACOBI blocks: the reduced rhs from k_schur MODE 1 over the long tiles alone
    "identity_precond": dict(scene=dict(model=PINHOLE, seed=65), filler=24, short=0, imask=0x061,
                             options=dict(preconditioner_type=_abi.PRECOND_IDENTITY)),
    "huber_const": dict(scene=dict(model=PINHOLE, shared_intrinsics=False, seed=66), filler=24, short=300, imask=0x061,
                        modify=_constants_and_outliers, loss=_abi.LOSS_HUBER),
}


def _problem(name):
    s = SCENES[name]
    p = long_track_scene(filler=s["filler"], short=s["short"], **s["scene"])
    if "modify" in s:
        s["modify"](p)
    return p


def _opts(mod, s, **kw):
    o = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, loss_function_type=s.get("loss", _abi.LOSS_TRIVIAL),
             robust_loss_width=2.0, intrinsics_to_optimize=s["scene"].get("intrinsics_to_optimize", FOCAL_RADIAL))
    o.update(s.get("options", {}))
    o.update(kw)
    return mod.default_options(**o)


def _check_layout(p, pk, s):
    """The long-tile layouts this file exists for, read from the host pack."""
    assert pk["rc"] == 0 and pk["imask"] == s["imask"], hex(pk["imask"])
    assert p.n_obs <= 50_000
    long_tile = (pk["tile_flags"] & 1) == 1
    tile, start, n = packed_extents(pk)
    end = start + n
    lng = long_tile[tile]
    assert np.array_equal(lng, n > 32)
    npts = np.diff(pk["tile_pt_begin"])
    used = np.bincount(tile, weights=n, minlength=pk["n_tiles"])
    assert (long_tile & (npts == 1) & (used == 256)).any(), "a long tile holding one 256-observation point"
    assert (long_tile & (npts == 1) & (used == 255)).any(), "a long tile holding one 255-observation point and a padding slot"
    assert (lng & (start % 32 != 0) & ((end - 1) // 32 - start // 32 >= 2)).any(), "a point from mid-warp over >= 3 warp slices"
    for e in (64, 96, 128, 65, 97, 129):
        assert (lng & (end == e)).any(), "a long point ending at slot %d of its tile" % e
    assert (long_tile & (npts == 7)).any(), "a long tile with seven points"
    if not s["scene"].get("shared_intrinsics", True):
        assert (pk["tile_nruns"] == 256).any(), "a tile of 256 (point, group) runs"
    if s["short"] == 0:
        assert long_tile.all(), "no normal tiles: the long kernels start at tile 0"
    else:
        assert not long_tile.all() and long_tile.any()


@pytest.fixture(scope="module")
def eng(request):
    if request.config.getoption("--mock-engine"):
        pytest.skip("per-block parity on long tiles: the real engine or its emulation build only")
    e = engine.Engine()
    yield e
    e.close()


STEPS = ((_abi.VEC_STEP_CAM, 6), (_abi.VEC_STEP_INTR, 10), (_abi.VEC_STEP_PT, 4))


def _expect(a, b, width, tol, what, floor=None):
    e, k = block_err(a, b, width, floor)
    assert e <= tol, "%s: block %d, error %.3g > %.0e" % (what, k, e, tol)


@pytest.mark.parametrize("name", list(SCENES))
def test_long_tiles_stage_parity(eng, oracle, name):
    s = SCENES[name]
    p = _problem(name)
    _check_layout(p, engine.debug_pack(p), s)
    opts_g = _opts(engine, s)
    eng.upload(p.copy(), opts_g)
    o = oracle.Oracle(p.copy(), _opts(oracle, s))
    ok_o, cost_o = o.linearize()
    ok_g, cost_g = eng.linearize()
    assert ok_o and ok_g
    assert abs(cost_g - cost_o) <= 1e-12 * cost_o
    lin_tol = 1e-10 if s.get("ext") else 1e-11  # dual-number evaluation of the EXT models (test_xx_camera_models_gpu)
    # residuals round relative to the pixel coordinates they are differences of (test_x_stream_ranges_gpu)
    _expect(eng.read(_abi.VEC_RESIDUALS), o.read(_abi.VEC_RESIDUALS), 2, lin_tol, "residuals", floor=np.abs(p.obs_xy).max(axis=1))
    for which, width in ((_abi.VEC_GRADIENT_CAM, 6), (_abi.VEC_GRADIENT_INTR, 10), (_abi.VEC_GRADIENT_PT, 4),
                         (_abi.VEC_COLNORM2_CAM, 6), (_abi.VEC_COLNORM2_INTR, 10), (_abi.VEC_COLNORM2_PT, 4)):
        _expect(eng.read(which), o.read(which), width, lin_tol, "linearize %d" % which)
    seen_c = np.bincount(p.obs_cam, minlength=p.n_cam) > 0
    seen_g = np.bincount(p.cam_group[seen_c], minlength=p.n_group) > 0
    rng = np.random.default_rng(5)
    free_c, free_i = o.read(_abi.VEC_COLNORM2_CAM) > 0, o.read(_abi.VEC_COLNORM2_INTR) > 0
    xs = [(rng.normal(size=p.n_cam * 6) * free_c, rng.normal(size=p.n_group * 10) * free_i) for _ in range(2)]
    for radius in (1e4, 1e2):
        assert o.prepare_linear_system(radius) and eng.prepare_linear_system(radius)
        _expect(eng.read(_abi.VEC_SCHUR_RHS_CAM), o.read(_abi.VEC_SCHUR_RHS_CAM), 6, 1e-10, "rhs cam @%g" % radius)
        _expect(eng.read(_abi.VEC_SCHUR_RHS_INTR), o.read(_abi.VEC_SCHUR_RHS_INTR), 10, 1e-10, "rhs intr @%g" % radius)
        if opts_g.preconditioner_type == _abi.PRECOND_SCHUR_JACOBI:
            Mc_g, Mc_o = eng.read(_abi.VEC_PRECOND_CAM).reshape(-1, 36), o.read(_abi.VEC_PRECOND_CAM).reshape(-1, 36)
            Mi_g, Mi_o = eng.read(_abi.VEC_PRECOND_INTR).reshape(-1, 100), o.read(_abi.VEC_PRECOND_INTR).reshape(-1, 100)
            _expect(Mc_g[seen_c], Mc_o[seen_c], 36, 1e-8, "precond cam @%g" % radius)
            _expect(Mi_g[seen_g], Mi_o[seen_g], 100, 1e-7, "precond intr @%g" % radius)
        for i, (xc, xi) in enumerate(xs):
            yc_o, yi_o = o.schur_matvec(xc, xi)
            yc_g, yi_g = eng.schur_matvec(xc, xi)
            _expect(yc_g, yc_o, 6, 1e-10, "matvec %d cam @%g" % (i, radius))
            _expect(yi_g, yi_o, 10, 1e-9, "matvec %d intr @%g" % (i, radius))
        ok_o, it_o, mcc_o = o.solve_linear_system()
        ok_g, it_g, mcc_g = eng.solve_linear_system()
        assert ok_o and ok_g
        assert it_o == it_g, (radius, it_o, it_g)
        assert abs(mcc_g - mcc_o) <= 1e-9 * abs(mcc_o), radius
        for which, width in STEPS:
            _expect(eng.read(which), o.read(which), width, 1e-8, "step %d @%g" % (which, radius))
        ok_o, cand_o = o.evaluate_step()
        ok_g, cand_g = eng.evaluate_step()
        assert ok_o and ok_g and abs(cand_g - cand_o) <= 1e-9 * cand_o, radius
    o.close()


def test_long_tiles_full_solve(eng, oracle):
    """ITERATIVE_SCHUR for 15 iterations on the per-camera scene with a 256-run tile: the same trajectory as the oracle."""
    s = SCENES["radtan_per_camera"]
    p0 = _problem("radtan_per_camera")
    po, pg = p0.copy(), p0.copy()
    so = oracle.solve(po, _opts(oracle, s, max_num_iterations=15))
    sg = eng.solve(pg, _opts(engine, s, max_num_iterations=15))
    assert sg.rc == 0 and sg.success and so.success
    assert abs(sg.initial_cost - so.initial_cost) <= 1e-12 * so.initial_cost
    assert sg.num_iterations == so.num_iterations and sg.termination_type == so.termination_type, (sg.message, so.message)
    assert [i["linear_solver_iterations"] for i in sg.iterations] == [i["linear_solver_iterations"] for i in so.iterations]
    co, cg = so.costs, sg.costs
    n = min(len(co), 10)
    assert np.all(np.abs(cg[:n] - co[:n]) <= 1e-9 * co[:n])
    assert np.all(np.abs(cg - co) <= 1e-6 * co)
