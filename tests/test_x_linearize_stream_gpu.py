"""The streaming linearisation of the normal tiles (k_linearize_stream) against the tile-per-CTA kernel (k_linearize) on the same
upload: both evaluate every observation with the same linearize_obs_any, so J, the residuals and the per-point blocks Hpp / gp
of the normal tiles must be bit-identical; the camera gradient, column norms and cost are sums in a different order (1e-12
relative).  The scenes mix normal tiles with long tiles (tracks of 33..48 observations), which both paths hand to k_linearize.
The *_at_scale scenes are sized from the device (helpers.stream_sized_scene) so that every warp of the streaming kernel owns at
least 2 NS + 1 slices: its ring is refilled and the next slice's gathers are handed over in registers within every range."""
import os

import numpy as np
import pytest

from helpers import rel_err, stream_sized_scene, warp_slice_counts
from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu

SCENES = {
    "shared_pinhole": dict(model=_abi.MODEL_PINHOLE, shared_intrinsics=True),
    "shared_radtan_all": dict(model=_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, shared_intrinsics=True, intrinsics_to_optimize=_abi.INTR_ALL),
    "per_camera_radtan": dict(model=_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, shared_intrinsics=False),
    "per_camera_radtan_all": dict(model=_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, shared_intrinsics=False, intrinsics_to_optimize=_abi.INTR_ALL),
}
AT_SCALE = {"shared_pinhole_at_scale": "shared_pinhole", "per_camera_radtan_at_scale": "per_camera_radtan"}
TRACKS = (3, 7, 31, 32, 33, 48)


def _constants_and_outliers(p):
    """constant blocks and outliers for the robust branch"""
    p.ext_const[1] = _abi.EXT_ALL_CONST
    p.ext_const[2] = _abi.EXT_POSITION_CONST
    p.pt_const[[5, 17, 40]] = 1
    p.obs_xy[::37] += 40.0


def _scene(kw, geometry=None):
    """geometry (Engine.stream_launch): as many points as give k_linearize_stream 2 NS + 1 slices per warp"""
    if geometry is not None:
        return stream_sized_scene(geometry, "linearize", lambda ns: 2 * ns + 1, track_lengths=TRACKS, modify=_constants_and_outliers,
                                  n_cam=120, obs_per_pt=48, seed=43, **kw)[0]
    p = synthetic.make_scene(n_cam=120, n_pt=260, obs_per_pt=48, seed=43, **kw)
    rng = np.random.default_rng(2)
    target = rng.choice(TRACKS, size=p.n_pt)
    seen = np.zeros(p.n_pt, int)
    keep = np.ones(p.n_obs, bool)
    for i in range(p.n_obs):
        q = int(p.obs_pt[i])
        seen[q] += 1
        keep[i] = seen[q] <= target[q]
    p = _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const,
                     p.obs_cam[keep], p.obs_pt[keep], p.obs_xy[keep])
    _constants_and_outliers(p)
    return p


@pytest.mark.parametrize("name", list(SCENES) + list(AT_SCALE))
def test_streaming_linearisation_matches_the_tile_kernel(request, name):
    if request.config.getoption("--mock-engine"):
        pytest.skip("raw device buffers: the real engine or its emulation build only")
    kw = SCENES[AT_SCALE.get(name, name)]
    eng = engine.Engine()
    try:
        opts = engine.default_options(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, loss_function_type=_abi.LOSS_HUBER,
                                      robust_loss_width=2.0,
                                      intrinsics_to_optimize=kw.get("intrinsics_to_optimize", _abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION))
        p = _scene(kw)
        if name in AT_SCALE:
            eng.upload(p, opts)
            p = _scene(kw, eng.stream_launch())
        pk = engine.debug_pack(p)
        flags = pk["tile_flags"]
        assert (flags & 1).any() and not (flags & 1).all(), "the scene must have normal and long tiles"
        eng.upload(p, opts)
        if name in AT_SCALE:
            g = eng.stream_launch()
            lin = g["linearize"]
            counts = warp_slice_counts(g["n_slices"], lin["grid"], lin["NW"])
            print("\n%s: n_sm %d, %d observations, %d normal slices, k_linearize_stream GW %d, slices per warp %d..%d"
                  % (name, g["n_sm"], p.n_obs, g["n_slices"], lin["grid"] * lin["NW"], counts.min(), counts.max()))
            assert lin["grid"] == g["n_sm"] and counts.min() >= 2 * lin["NS"] + 1
        a = eng.linearize_raw(tile_kernel=False)
        b = eng.linearize_raw(tile_kernel=True)
    finally:
        eng.close()
    assert a["failed"] == 0.0 and b["failed"] == 0.0
    assert np.abs(a["J"]).max() > 0.0
    # The emulation build with FMA contraction (TBA_EMU_LIBNAME) rounds its own way: the streaming kernel pins two J_l entries
    # to the rounding nvcc gives k_linearize, and g++ contracts differently.
    exact = "TBA_EMU_LIBNAME" not in os.environ
    # points of the long tiles are summed across warps with shared-memory atomics (in no fixed order) by k_linearize in both runs
    begin = pk["tile_pt_begin"]
    normal = np.zeros(len(a["Hpp"]), bool)
    for t in np.nonzero((flags & 1) == 0)[0]:
        normal[begin[t]:begin[t + 1]] = True
    assert normal.any() and not normal.all()
    for k, sel in (("J", slice(None)), ("res", slice(None)), ("Hpp", normal), ("gp", normal)):
        if exact:
            assert np.array_equal(a[k][sel], b[k][sel]), k
        else:
            assert rel_err(a[k][sel], b[k][sel]) < 1e-15, k
    for k in ("Hpp", "gp"):
        assert rel_err(a[k][~normal], b[k][~normal]) < 1e-12, k
    for k in ("g", "cn"):
        assert rel_err(a[k], b[k]) < 1e-12, k
    assert abs(a["cost"] - b["cost"]) <= 1e-12 * b["cost"]
    assert abs(a["fixed"] - b["fixed"]) <= 1e-12 * b["fixed"]
