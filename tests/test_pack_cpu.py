"""Host-side packing (theiasfm_b200/csrc/tba_pack.h, the code tba_upload runs) checked on CPU through tba_debug_pack:
every observation lands in exactly one slot, points are contiguous, a short track never straddles a warp slice,
long tracks live in long tiles, runs / flags / masks follow the rules of DESIGN.md section 4."""
import numpy as np
import pytest

from helpers import exact_tracks
from theiasfm_b200 import _abi, engine, synthetic


def _ragged_scene(seed=3, n_groups_mode="shared"):
    p = synthetic.make_scene(n_cam=90, n_pt=700, obs_per_pt=40, seed=seed, shared_intrinsics=(n_groups_mode == "shared"))
    rng = np.random.default_rng(seed)
    target = rng.choice([1, 2, 5, 9, 17, 31, 32, 33, 40], size=p.n_pt)
    target[11] = 0  # a point without observations
    seen = np.zeros(p.n_pt, int)
    keep = np.zeros(p.n_obs, bool)
    for i in range(p.n_obs):
        q = p.obs_pt[i]
        seen[q] += 1
        keep[i] = seen[q] <= target[q]
    perm = rng.permutation(int(keep.sum()))
    cam_group = p.cam_group.copy()
    group_model, intr, gmask = p.group_model, p.intr, p.group_const_mask
    if n_groups_mode == "few":  # 3 shared groups
        cam_group = (np.arange(p.n_cam) % 3).astype(np.int32)
        group_model, intr, gmask = p.group_model[:3], p.intr[:3], p.group_const_mask[:3]
    q = _abi.Problem(p.ext, p.ext_const, cam_group, group_model, intr, gmask, p.pt, p.pt_const,
                     p.obs_cam[keep][perm], p.obs_pt[keep][perm], p.obs_xy[keep][perm])
    q.ext_const[5] = _abi.EXT_ALL_CONST
    q.pt_const[[3, 4]] = 1
    return q


LONG_TRACKS = {
    "track_256": [256],                 # 256 per-camera groups: 256 runs, the most a point (and a tile) can have
    "track_256_repeat": [256],          # the same track with one camera observing the point twice: 255 runs
    "track_255": [255],                 # a padding slot behind it
    "long_33_36": [33] * 7 + [36] * 7,  # two long tiles of seven points each
}


def _long_scene(mode, seed=7):
    """Long tracks over per-camera intrinsics groups (a point has one run per distinct camera), a few short ones, observations in
    random order."""
    lengths = LONG_TRACKS[mode] + [2, 9, 32]
    p = synthetic.make_scene(n_cam=260, n_pt=len(lengths) + 8, obs_per_pt=max(lengths), seed=seed, shared_intrinsics=False)
    p = exact_tracks(p, lengths)
    if mode == "track_256_repeat":
        o = np.nonzero(p.obs_pt == 0)[0]
        p.obs_cam[o[100]] = p.obs_cam[o[7]]
    perm = np.random.default_rng(seed).permutation(p.n_obs)
    q = _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const,
                     p.obs_cam[perm], p.obs_pt[perm], p.obs_xy[perm])
    q.ext_const[5] = _abi.EXT_ALL_CONST
    q.pt_const[[1, len(lengths) - 1]] = 1
    return q


@pytest.mark.parametrize("mode", ["shared", "per_camera", "few"] + list(LONG_TRACKS))
def test_pack_invariants(mode):
    p = _long_scene(mode) if mode in LONG_TRACKS else _ragged_scene(seed=7, n_groups_mode=mode)
    k = engine.debug_pack(p)
    assert k["rc"] == 0
    n_slots, n_tiles = k["n_slots"], k["n_tiles"]
    assert n_slots == n_tiles * 256
    valid = k["slot_cam"] >= 0
    counts = np.bincount(p.obs_pt, minlength=p.n_pt)
    # 1. a bijection between observations and valid slots, carrying the right camera / point / measurement
    orig = k["slot_orig"][valid]
    assert valid.sum() == p.n_obs and np.array_equal(np.sort(orig), np.arange(p.n_obs))
    assert (k["slot_orig"][~valid] == -1).all()
    assert np.array_equal(k["slot_cam"][valid], p.obs_cam[orig])
    assert np.array_equal(k["pk2caller"][k["slot_pt"][valid]], p.obs_pt[orig])
    s = np.nonzero(valid)[0]
    wq, lane = s // 32, s % 32
    assert np.array_equal(k["xy"][(wq * 2 + 0) * 32 + lane], p.obs_xy[orig, 0])
    assert np.array_equal(k["xy"][(wq * 2 + 1) * 32 + lane], p.obs_xy[orig, 1])
    # 2. packed points: exactly the points with observations; short tracks first (caller order), then long tracks
    pk = k["pk2caller"]
    assert set(pk.tolist()) == set(np.nonzero(counts > 0)[0].tolist()) and len(set(pk.tolist())) == len(pk)
    n_short = int(((counts > 0) & (counts <= 32)).sum())
    assert np.array_equal(pk[:n_short], np.nonzero((counts > 0) & (counts <= 32))[0])
    assert np.array_equal(pk[n_short:], np.nonzero(counts > 32)[0]) and k["n_long_points"] == int((counts > 32).sum())
    # 3. per packed point: contiguous slots, inside one tile; short tracks inside one warp slice of a normal tile,
    #    long tracks in long tiles; (group, camera, observation index) order inside the point
    tb = k["tile_pt_begin"]
    assert tb[0] == 0 and tb[-1] == len(pk) and (np.diff(tb) > 0).all() and (np.diff(tb) <= 256).all()
    for kp in range(len(pk)):
        sl = np.nonzero(valid & (k["slot_pt"] == kp))[0]
        assert len(sl) == counts[pk[kp]] and (np.diff(sl) == 1).all()
        t = sl[0] // 256
        assert sl[-1] // 256 == t and tb[t] <= kp < tb[t + 1]
        if counts[pk[kp]] <= 32:
            assert k["tile_flags"][t] == 0 and sl[0] // 32 == sl[-1] // 32
        else:
            assert k["tile_flags"][t] == 1
        cams = k["slot_cam"][sl]
        key = np.diff(p.cam_group[cams].astype(np.int64) * 100000 + cams)
        assert ((key > 0) | ((key == 0) & (np.diff(k["slot_orig"][sl]) > 0))).all()
    # 4. runs: a new run whenever (point, group) changes, numbered from 0 inside each tile
    for t in range(n_tiles):
        sl = np.arange(t * 256, (t + 1) * 256)
        sl = sl[valid[sl]]
        keys = list(zip(k["slot_pt"][sl].tolist(), p.cam_group[k["slot_cam"][sl]].tolist()))
        run, last, expect = -1, None, []
        for kk in keys:
            if kk != last:
                run += 1
                last = kk
            expect.append(run)
        assert k["slot_run"][sl].tolist() == expect and k["tile_nruns"][t] == run + 1
    assert (k["slot_run"][~valid] == -1).all()
    # 5. masks and the "all blocks constant" flag
    cam_cnt = np.bincount(p.obs_cam, minlength=p.n_cam)
    grp_cnt = np.bincount(p.cam_group, weights=cam_cnt, minlength=p.n_group)
    mask = k["mask"]
    for c in range(p.n_cam):
        exp = np.zeros(6)
        if cam_cnt[c] > 0:
            exp[:3] = 0 if p.ext_const[c] & _abi.EXT_POSITION_CONST else 1
            exp[3:] = 0 if p.ext_const[c] & _abi.EXT_ORIENTATION_CONST else 1
        assert np.array_equal(mask[c * 6:c * 6 + 6], exp)
    for g in range(p.n_group):
        K = _abi.MODEL_NUM_PARAMS[int(p.group_model[g])]
        exp = np.array([1.0 if (j < K and grp_cnt[g] > 0 and not (int(p.group_const_mask[g]) >> j) & 1) else 0.0 for j in range(10)])
        assert np.array_equal(mask[p.n_cam * 6 + g * 10:p.n_cam * 6 + g * 10 + 10], exp)
    cam_free = mask[:p.n_cam * 6].reshape(-1, 6).any(axis=1)
    grp_free = mask[p.n_cam * 6:].reshape(-1, 10).any(axis=1)
    cams = k["slot_cam"][valid]
    exp_fixed = ~(cam_free[cams] | grp_free[p.cam_group[cams]] | (p.pt_const[pk[k["slot_pt"][valid]]] == 0))
    assert np.array_equal(k["slot_flags"][valid].astype(bool), exp_fixed)
    assert k["NI"] == 3 and k["imask"] == 0x61  # default mask: f, k1, k2


def test_pack_column_set_selection_and_limits():
    base = synthetic.make_scene(n_cam=20, n_pt=100, obs_per_pt=5, seed=1)
    for flags, model, imask in ((_abi.INTR_NONE, 0, 0x000), (_abi.INTR_FOCAL_LENGTH, 0, 0x001),
                                (_abi.INTR_FOCAL_LENGTH | _abi.INTR_RADIAL_DISTORTION, 1, 0x0E1), (_abi.INTR_ALL, 0, 0x07F),
                                (_abi.INTR_ALL, 1, 0x3FF), (_abi.INTR_FOCAL_LENGTH | _abi.INTR_PRINCIPAL_POINTS, 0, 0x07F),
                                (_abi.INTR_TANGENTIAL_DISTORTION, 1, 0x3FF)):
        p = synthetic.make_scene(n_cam=20, n_pt=100, obs_per_pt=5, seed=1, model=model, intrinsics_to_optimize=flags)
        assert engine.debug_pack(p)["imask"] == imask, (flags, model)
    # padding of a regular L = 10 scene: 3 points per warp slice -> 30/32 slots used
    p = synthetic.make_scene(n_cam=50, n_pt=2400, obs_per_pt=10, seed=2)
    k = engine.debug_pack(p)
    assert k["n_slots"] == 2400 * 10 // 240 * 256 and k["n_long_points"] == 0
    # out-of-range indices and over-long tracks are refused
    bad = base.copy(); bad.obs_cam[3] = 999
    assert engine.debug_pack(bad)["rc"] == _abi.ERR_INVALID_ARGUMENT
    long_ = synthetic.make_scene(n_cam=600, n_pt=3, obs_per_pt=290, seed=1)
    assert engine.debug_pack(long_)["rc"] == _abi.ERR_UNSUPPORTED


def test_scattered_observation_order_packs_like_the_grouped_one():
    """Observations that are NOT grouped by point (the adapter flattens per view: bundle_adjuster.cc:125-134) take the two-level counting
    sort of pack_count_and_sort (buckets of points, no contended atomics) instead of the run-based path: the packed problem -- tiles,
    slot cameras / points / measurements -- must be the same as for the point-grouped order of the same observations, and every slot must
    still name its caller observation."""
    _check_scattered_equals_grouped(synthetic.make_scene(n_cam=40, n_pt=6000, obs_per_pt=7, seed=21, shared_intrinsics=False))


def test_scattered_order_with_many_points_and_parallel_prefix():
    """150 k points: several chunks in the parallel prefix sum / packed-point list, point buckets of more than one point (shift > 0)."""
    _check_scattered_equals_grouped(synthetic.make_scene(n_cam=12, n_pt=150_000, obs_per_pt=3, seed=22))


def _check_scattered_equals_grouped(p):
    p.pt_const[::9] = 1
    rng = np.random.default_rng(5)
    by_view = np.argsort(p.obs_cam, kind="stable")
    shuffled = rng.permutation(p.n_obs)
    base = engine.debug_pack(p)
    assert base["rc"] == 0
    for perm in (by_view, shuffled):
        q = _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const,
                         p.obs_cam[perm].copy(), p.obs_pt[perm].copy(), p.obs_xy[perm].copy())
        k = engine.debug_pack(q)
        assert k["rc"] == 0 and k["n_slots"] == base["n_slots"] and k["n_tiles"] == base["n_tiles"]
        for name in ("slot_cam", "slot_pt", "slot_run", "slot_flags", "xy", "pk2caller", "tile_pt_begin", "tile_nruns", "tile_flags", "mask"):
            assert np.array_equal(k[name], base[name]), name
        valid = k["slot_cam"] >= 0
        orig = k["slot_orig"][valid]
        assert np.array_equal(np.sort(orig), np.arange(p.n_obs))
        assert np.array_equal(q.obs_cam[orig], k["slot_cam"][valid]) and np.array_equal(perm[orig], base["slot_orig"][valid])


def test_worker_pool_stress(tmp_path):
    """tests/host_pack_pool.cc: concurrent callers, nested loops, exact results through the pack's worker pool and its fall-back."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "host_pack_pool")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", "-I" + os.path.join(root, "include"), "-o", exe, os.path.join(root, "tests", "host_pack_pool.cc")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "pack pool ok" in out.stdout, out.stdout + out.stderr
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300, env=dict(os.environ, TBA_PACK_POOL="0"))
    assert out.returncode == 0 and "pack pool ok" in out.stdout
