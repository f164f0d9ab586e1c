"""Stage parity of the persistent warp-slice kernels (k_linearize_stream, k_prepare_stream, k_schur_stream MODE 0 / 1 / 2) when
their warps own many slices.

Warp gw of GW = grid * NW owns the slices [n*gw/GW, n*(gw+1)/GW) of the normal tiles and pipelines them through an NS-stage
TMA / mbarrier ring: stage s is refilled with slice s + NS, the gathers of slice s + 1 are handed over in registers, and the
shared-group sums stay in registers over the whole range.  The grid is capped at one CTA per SM, so below n_sm * NW slices every
warp owns at most one slice and none of that runs.  Here the scenes are sized from the device's launch geometry
(Engine.stream_launch) to given slice counts per warp: the cap just binding, one tile above it, NS, NS + 1 (the first refill),
2 NS + 1 and more (the ring's parity back at 0, accumulators over many slices), and a count that alternates between the floor and
the ceiling.  Each scene walks one LM iteration against the oracle stage by stage and compares every camera, group, point and
observation block on its own (helpers.block_err): a slice dropped from or repeated in a range moves only the blocks it touches."""
import numpy as np
import pytest

from helpers import STREAM_KERNELS, block_err, stream_sized_scene, warp_slice_counts
from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu

PINHOLE, RADTAN, FISHEYE = _abi.MODEL_PINHOLE, _abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, _abi.MODEL_FISHEYE
FOCAL_RADIAL = _abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION


def _constants_and_outliers(p):
    p.ext_const[1] = _abi.EXT_ALL_CONST
    p.ext_const[2] = _abi.EXT_POSITION_CONST
    p.ext_const[3] = _abi.EXT_ORIENTATION_CONST
    p.pt_const[[q for q in (5, 17, 40) if q < p.n_pt]] = 1
    p.obs_xy[::37] += 40.0  # outliers for the robust branch


# scene: make_scene arguments; imask: the intrinsics column set the engine must dispatch
SCENES = {
    "pinhole_huber_const": dict(scene=dict(n_cam=64, obs_per_pt=6, model=PINHOLE, seed=51, intrinsics_to_optimize=_abi.INTR_FOCAL_LENGTH),
                                imask=0x001, modify=_constants_and_outliers, loss=_abi.LOSS_HUBER),
    "radtan_per_camera": dict(scene=dict(n_cam=48, obs_per_pt=6, model=RADTAN, shared_intrinsics=False, seed=52), imask=0x0E1),
    "radtan_shared_all": dict(scene=dict(n_cam=48, obs_per_pt=6, model=RADTAN, seed=53, intrinsics_to_optimize=_abi.INTR_ALL), imask=0x3FF),
    "pinhole_none": dict(scene=dict(n_cam=48, obs_per_pt=5, model=PINHOLE, seed=54, intrinsics_to_optimize=_abi.INTR_NONE), imask=0x000),
    "pinhole_focal_radial": dict(scene=dict(n_cam=48, obs_per_pt=7, model=PINHOLE, seed=55, intrinsics_to_optimize=FOCAL_RADIAL), imask=0x061),
    "pinhole_all": dict(scene=dict(n_cam=48, obs_per_pt=6, model=PINHOLE, seed=56, intrinsics_to_optimize=_abi.INTR_ALL), imask=0x07F),
    # tracks cut to 3..48 observations: long tiles (k_linearize / k_schur / k_precond_* from the first long tile) after the normal ones
    "long_short": dict(scene=dict(n_cam=120, obs_per_pt=48, model=PINHOLE, seed=57), track_lengths=(3, 7, 31, 32, 33, 48),
                       imask=0x061, modify=_constants_and_outliers, loss=_abi.LOSS_HUBER),
    # no SCHUR_JACOBI blocks: the reduced rhs comes from k_schur_stream MODE 1 instead of k_prepare_stream
    "identity_precond": dict(scene=dict(n_cam=48, obs_per_pt=6, model=PINHOLE, seed=58), imask=0x061,
                             options=dict(preconditioner_type=_abi.PRECOND_IDENTITY)),
    # EXT camera model: every tile through k_linearize<0x3FF, true>, the streaming prepare and matvec at 0x3FF
    "fisheye_shared": dict(scene=dict(n_cam=48, obs_per_pt=6, model=FISHEYE, seed=59), imask=0x3FF, ext=True),
}

# slices per warp of the kernel the scene is sized for, as a function of its ring depth NS, and slices added on top
REGIMES = {
    "cap": (lambda ns: 1, 0),            # n_slices = n_sm * NW (rounded up to a tile): the grid cap just binds
    "cap_plus_tile": (lambda ns: 1, 8),  # one tile more: a few warps own 2
    "ns": (lambda ns: ns, 0),            # the ring filled once, never refilled
    "ns_plus_1": (lambda ns: ns + 1, 0), # the first refill
    "many": (lambda ns: 2 * ns + 1, 0),  # the barrier parity back at 0; accumulators over many slices
    "mixed": (lambda ns: ns + 0.5, 0),   # n mod GW = GW / 2: floor and ceiling ranges alternate
}

CASES = [("pinhole_huber_const", k, r) for r in REGIMES for k in STREAM_KERNELS]
CASES += [("radtan_per_camera", "matvec", "mixed")]
CASES += [(s, None, "many") for s in SCENES]


@pytest.fixture(scope="module")
def eng(request):
    if request.config.getoption("--mock-engine"):
        pytest.skip("launch geometry and per-block parity: the real engine or its emulation build only")
    e = engine.Engine()
    yield e
    e.close()


def _opts(mod, scene):
    kw = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, loss_function_type=scene.get("loss", _abi.LOSS_TRIVIAL),
              robust_loss_width=2.0, intrinsics_to_optimize=scene["scene"].get("intrinsics_to_optimize", FOCAL_RADIAL))
    kw.update(scene.get("options", {}))
    return mod.default_options(**kw)


_GEOMETRY = {}


def _geometry(eng, name):
    """Engine.stream_launch of a small version of the scene: the device's SM count and the warps / stages of each kernel at the
    scene's intrinsics instantiation."""
    if name not in _GEOMETRY:
        s = SCENES[name]
        eng.upload(synthetic.make_scene(n_pt=200, **s["scene"]), _opts(engine, s))
        _GEOMETRY[name] = eng.stream_launch()
    return _GEOMETRY[name]


def _used(geo, options):
    """The streaming kernels this upload runs."""
    used = {"linearize": not geo["has_ext_models"], "prepare": options.preconditioner_type != _abi.PRECOND_IDENTITY,
            "matvec": True, "rhs_backsub": True}
    return [k for k in STREAM_KERNELS if used[k]]


def _check_regime(counts, geo_k, n_sm, regime):
    ns = geo_k["NS"]
    GW = geo_k["grid"] * geo_k["NW"]
    n = int(counts.sum())
    vals, hits = np.unique(counts, return_counts=True)
    if regime == "cap":
        assert geo_k["grid"] == n_sm and counts.min() == 1 and counts.max() <= 2 and (counts == 2).sum() == n - GW < 8
    elif regime == "cap_plus_tile":
        assert geo_k["grid"] == n_sm and counts.min() >= 1 and counts.max() >= 2 and n - GW >= 8
    elif regime in ("ns", "ns_plus_1"):
        want = ns if regime == "ns" else ns + 1
        assert counts.min() >= want and (counts == want).sum() > GW // 2
    elif regime == "many":
        assert counts.min() >= 2 * ns + 1
    else:
        if n % GW == 0:
            pytest.skip("GW = %d warps: no whole number of tiles near %d slices per warp splits unevenly" % (GW, n // GW))
        assert len(vals) == 2 and vals[1] == vals[0] + 1 and vals[0] >= ns and hits.min() >= GW // 4


STEPS = ((_abi.VEC_STEP_CAM, 6), (_abi.VEC_STEP_INTR, 10), (_abi.VEC_STEP_PT, 4))


def _expect(a, b, width, tol, what, floor=None):
    e, k = block_err(a, b, width, floor)
    assert e <= tol, "%s: block %d, error %.3g > %.0e" % (what, k, e, tol)


@pytest.mark.parametrize("name,kernel,regime", CASES)
def test_stream_ranges_stage_parity(eng, oracle, name, kernel, regime):
    s = SCENES[name]
    geo = _geometry(eng, name)
    p, pk = stream_sized_scene(geo, kernel, REGIMES[regime][0], extra_slices=REGIMES[regime][1], track_lengths=s.get("track_lengths"),
                               modify=s.get("modify"), **s["scene"])
    assert pk["imask"] == s["imask"], hex(pk["imask"])
    opts_g = _opts(engine, s)
    eng.upload(p.copy(), opts_g)
    g = eng.stream_launch()
    assert g["imask"] == s["imask"] and g["has_ext_models"] == s.get("ext", False)
    assert g["n_slices"] == 8 * int(((pk["tile_flags"] & 1) == 0).sum())
    if "track_lengths" in s:
        assert (pk["tile_flags"] & 1).any(), "the scene must have long tiles"
    used = _used(g, opts_g)
    if kernel is not None and kernel not in used:
        pytest.skip("%s does not run for this scene" % kernel)
    if kernel == "rhs_backsub" and (g["rhs_backsub"]["NW"], g["rhs_backsub"]["NS"]) == (g["matvec"]["NW"], g["matvec"]["NS"]):
        pytest.skip("k_schur_stream MODE 1 / 2 has the matvec's launch geometry here: the matvec case sizes the same scene")
    counts = {k: warp_slice_counts(g["n_slices"], g[k]["grid"], g[k]["NW"]) for k in used}
    print("\n%s %s %s: n_sm %d, %d observations, %d normal slices; slices per warp: %s" % (
        name, kernel or "all", regime, g["n_sm"], p.n_obs, g["n_slices"],
        "; ".join("%s (GW %d, NS %d) %s" % (k, g[k]["grid"] * g[k]["NW"], g[k]["NS"],
                                             dict(zip(*(v.tolist() for v in np.unique(c, return_counts=True)))))
                  for k, c in counts.items())))
    for k in ([kernel] if kernel is not None else used):
        _check_regime(counts[k], g[k], g["n_sm"], regime)

    o = oracle.Oracle(p.copy(), _opts(oracle, s))
    ok_o, cost_o = o.linearize()
    ok_g, cost_g = eng.linearize()
    assert ok_o and ok_g
    assert abs(cost_g - cost_o) <= 1e-12 * cost_o
    lin_tol = 1e-10 if s.get("ext") else 1e-11  # dual-number evaluation of the EXT models (test_xx_camera_models_gpu)
    # a residual is the difference of a ~500 px projection and the observation: it rounds relative to the pixel coordinates, not
    # to itself (a 0.06 px residual differed by 5e-12 of its size under emulation)
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
            # blocks of observed cameras / groups only: for a camera without observations (a scene of a few tiles) the engine
            # stores an identity block where the oracle inverts the bare LM diagonal; its rhs is 0, so no PCG iterate moves it
            Mc_g, Mc_o = eng.read(_abi.VEC_PRECOND_CAM).reshape(-1, 36), o.read(_abi.VEC_PRECOND_CAM).reshape(-1, 36)
            Mi_g, Mi_o = eng.read(_abi.VEC_PRECOND_INTR).reshape(-1, 100), o.read(_abi.VEC_PRECOND_INTR).reshape(-1, 100)
            _expect(Mc_g[seen_c], Mc_o[seen_c], 36, 1e-8, "precond cam @%g" % radius)
            _expect(Mi_g[seen_g], Mi_o[seen_g], 100, 1e-7, "precond intr @%g" % radius)
        for i, (xc, xi) in enumerate(xs):
            yc_o, yi_o = o.schur_matvec(xc, xi)
            yc_g, yi_g = eng.schur_matvec(xc, xi)
            _expect(yc_g, yc_o, 6, 1e-10, "matvec %d cam @%g" % (i, radius))
            # an intrinsics row of S sums the Schur complement over every observation of the group, and the sum cancels: with a
            # random x a shared group's |y| came out at 1e-2 of its terms, and 1.1e-10 relative (9e-13 absolute) under emulation.
            # A slice missing from a range moves the block by its share of the terms, orders of magnitude more.
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
