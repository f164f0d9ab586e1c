"""Shared helpers for the parity tests."""
import os

import numpy as np

from theiasfm_b200 import _abi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reprojection_golden.npz")


def golden_problem(ext=False):
    """All golden cases as ONE problem: case i = camera i, group i, point i, observation i.  ext=True: the FISHEYE / FOV /
    DIVISION_UNDISTORTION vectors (reprojection_golden_ext.npz)."""
    g = np.load(GOLDEN.replace("reprojection_golden.npz", "reprojection_golden_ext.npz") if ext else GOLDEN)
    n = len(g["model"])
    prob = _abi.Problem(g["ext"], np.zeros(n, np.uint8), np.arange(n, dtype=np.int32), g["model"], g["intr"],
                        np.zeros(n, np.uint32), g["pt"], np.zeros(n, np.uint8), np.arange(n, dtype=np.int32),
                        np.arange(n, dtype=np.int32), g["xy"])
    return prob, g


def rel_err(a, b):
    a = np.asarray(a, float); b = np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(1e-300, np.max(np.abs(b))))


def block_err(a, b, width, floor=None):
    """Per-block relative error of a against the reference b, blocks of `width` consecutive entries (a camera, a group, a point, an
    observation): max|a - b| over the block divided by max(max|b_block|, 1e-6 max|b|) -- and by at least floor[block] if given.
    A block where b is exactly zero must be exactly zero in a as well (constant blocks, masked coordinates), else its error is
    inf.  Returns (largest error, its block)."""
    a = np.asarray(a, float).reshape(-1, width); b = np.asarray(b, float).reshape(-1, width)
    if len(b) == 0:
        return 0.0, -1
    d, s = np.abs(a - b).max(axis=1), np.abs(b).max(axis=1)
    den = np.maximum(s, 1e-6 * s.max() if s.max() > 0 else 1.0)
    if floor is not None:
        den = np.maximum(den, floor)
    err = np.where(s == 0, np.where(np.abs(a).max(axis=1) == 0, 0.0, np.inf), d / den)
    k = int(np.argmax(err))
    return float(err[k]), k


def warp_slice_counts(n_slices, grid, nw):
    """Slices per warp of a persistent warp-slice kernel: warp gw of GW = grid * nw owns [n_slices*gw/GW, n_slices*(gw+1)/GW)."""
    GW = grid * nw
    return np.diff(n_slices * np.arange(GW + 1, dtype=np.int64) // GW)


def cut_tracks(p, lengths, seed=1):
    """Every track keeps its first n observations, n drawn from `lengths` per point."""
    target = np.random.default_rng(seed).choice(lengths, size=p.n_pt)
    order = np.argsort(p.obs_pt, kind="stable")
    q = p.obs_pt[order]
    first = np.searchsorted(q, q)  # index of the first observation of the same point in the sorted order
    keep = np.zeros(p.n_obs, bool)
    keep[order] = np.arange(p.n_obs) - first < target[q]
    return _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt, p.pt_const,
                        p.obs_cam[keep], p.obs_pt[keep], p.obs_xy[keep])


def exact_tracks(p, lengths):
    """Point i of the result is a track of exactly lengths[i] observations: the first lengths[i] observations of the next point
    of p, in caller order, that has at least that many.  Long tracks are packed into long tiles in caller order, so the list
    fixes the long-tile layout."""
    order = np.argsort(p.obs_pt, kind="stable")
    counts = np.bincount(p.obs_pt, minlength=p.n_pt)
    begin = np.concatenate([[0], np.cumsum(counts)])
    src, q = [], 0
    for n in lengths:
        while q < p.n_pt and counts[q] < n:
            q += 1
        assert q < p.n_pt, "the scene has too few points with %d observations" % n
        src.append(q)
        q += 1
    idx = np.concatenate([order[begin[q]:begin[q] + n] for q, n in zip(src, lengths)])
    return _abi.Problem(p.ext, p.ext_const, p.cam_group, p.group_model, p.intr, p.group_const_mask, p.pt[src], p.pt_const[src],
                        p.obs_cam[idx], np.repeat(np.arange(len(lengths), dtype=np.int32), lengths), p.obs_xy[idx])


# Long tracks in caller order and the long tiles they pack into (tile-relative slot ranges):
#   [0, 256)                                   one point fills the tile
#   [0, 255) + padding                         the largest point that leaves a padding slot
#   [0, 33) [33, 133) [133, 197)               a point from lane 1 of slice 1 over slices 1..4
#   [0, 96) [96, 129)                          ends on a warp boundary / one slot past one
#   [0, 128) [128, 256)
#   [0, 64) [64, 97) [97, 247)
#   [0, 65) [65, 255)
#   seven points of 36
LONG_LAYOUT = (256, 255, 33, 100, 64, 96, 33, 128, 128, 64, 33, 150, 65, 190) + (36,) * 7


def long_track_scene(seed, filler=24, short=0, n_cam=260, **scene_kw):
    """synthetic.make_scene(n_cam, seed=seed, **scene_kw) cut to the tracks LONG_LAYOUT, then `filler` more tracks of 33..256
    observations and `short` tracks of 2..32 (normal tiles), in that caller order.  A 256-observation track needs 256 cameras."""
    rng = np.random.default_rng(seed)
    lengths = list(LONG_LAYOUT) + rng.integers(33, 257, filler).tolist() + rng.integers(2, 33, short).tolist()
    from theiasfm_b200 import synthetic
    p = synthetic.make_scene(n_cam=n_cam, n_pt=len(lengths) + 40, obs_per_pt=256, seed=seed, **scene_kw)
    return exact_tracks(p, lengths)


def packed_extents(pk):
    """(tile, first slot inside the tile, observation count) of every packed point of the host packing pk (engine.debug_pack)."""
    valid = pk["slot_cam"] >= 0
    slots, kp = np.nonzero(valid)[0], pk["slot_pt"][valid]
    first = np.zeros(pk["n_packed_points"], np.int64)
    first[kp[::-1]] = slots[::-1]
    return first // 256, first % 256, np.bincount(kp, minlength=pk["n_packed_points"])


STREAM_KERNELS = ("linearize", "prepare", "matvec", "rhs_backsub")


def stream_target_slices(geometry, kernel, per_warp):
    """Normal-tile slice count (a multiple of 8, one tile) giving `kernel` of the launch geometry `geometry` (Engine.stream_launch)
    per_warp slices in most warps once its grid is capped at one CTA per SM; kernel None: the largest such count over the four.
    per_warp may be a function of the kernel's ring depth NS."""
    if kernel is None:
        return max(stream_target_slices(geometry, k, per_warp) for k in STREAM_KERNELS)
    if callable(per_warp):
        per_warp = per_warp(geometry[kernel]["NS"])
    GW = geometry["n_sm"] * geometry[kernel]["NW"]
    return max(8, -(-int(round(per_warp * GW)) // 8) * 8)


def normal_slices(p):
    """(slices of the normal tiles, the host packing) of a problem: what the streaming kernels partition among their warps."""
    from theiasfm_b200 import engine
    pk = engine.debug_pack(p)
    assert pk["rc"] == 0, pk["rc"]
    return 8 * int(((pk["tile_flags"] & 1) == 0).sum()), pk


def stream_sized_scene(geometry, kernel, per_warp, extra_slices=0, track_lengths=None, modify=None, **scene_kw):
    """A seeded synthetic.make_scene(**scene_kw) whose normal tiles hold exactly stream_target_slices(...) + extra_slices warp
    slices.  The point count is searched with the host packing (engine.debug_pack): tracks are cut to `track_lengths` and
    `modify(problem)` applied (constant blocks, outliers) before every packing.  Returns (problem, packing)."""
    from theiasfm_b200 import synthetic
    target = stream_target_slices(geometry, kernel, per_warp) + extra_slices

    def make(n_pt):
        p = synthetic.make_scene(n_pt=int(n_pt), **scene_kw)
        if track_lengths is not None:
            p = cut_tracks(p, track_lengths)
        if modify is not None:
            modify(p)
        return (p,) + normal_slices(p)

    n_pt, seen = 64, {}
    lo, hi = 0, None  # n_pt below / above the target
    for _ in range(60):
        p, s, pk = make(n_pt)
        seen[n_pt] = s
        if s == target:
            return p, pk
        if s < target:
            lo = max(lo, n_pt)
        else:
            hi = n_pt if hi is None else min(hi, n_pt)
        if hi is None:
            nxt = max(n_pt + 1, int(n_pt * target / max(s, 1) * 1.02))
        elif hi - lo <= 1:
            break
        else:  # interpolate inside the bracket, never on its ends
            s_lo = seen.get(lo, 0)
            nxt = lo + int(round((hi - lo) * (target - s_lo) / max(seen[hi] - s_lo, 1)))
            nxt = min(max(nxt, lo + 1), hi - 1)
        n_pt = nxt
    raise AssertionError("no point count packs to %d normal slices (tried %s)" % (target, sorted(seen.items())))


def free_masks(p):
    """(free_cam [n_cam,6], free_intr [n_group,10], free_pt [n_pt,4]) booleans."""
    fc = np.ones((p.n_cam, 6), bool)
    fc[:, :3] = (p.ext_const & _abi.EXT_POSITION_CONST)[:, None] == 0
    fc[:, 3:] = (p.ext_const & _abi.EXT_ORIENTATION_CONST)[:, None] == 0
    fi = np.zeros((p.n_group, 10), bool)
    for g in range(p.n_group):
        K = _abi.MODEL_NUM_PARAMS[int(p.group_model[g])]
        for j in range(K):
            fi[g, j] = not ((int(p.group_const_mask[g]) >> j) & 1)
    fp = np.repeat((p.pt_const == 0)[:, None], 4, axis=1)
    return fc, fi, fp


def dense_jacobian(p, J_obs):
    """Assemble the dense (masked, unscaled) Jacobian [2*n_obs, 6*n_cam + 10*n_group + 4*n_pt]."""
    fc, fi, fp = free_masks(p)
    nc, ng, npt, no = p.n_cam, p.n_group, p.n_pt, p.n_obs
    J = np.zeros((2 * no, 6 * nc + 10 * ng + 4 * npt))
    for k in range(no):
        c, q = int(p.obs_cam[k]), int(p.obs_pt[k]); g = int(p.cam_group[c])
        J[2 * k:2 * k + 2, 6 * c:6 * c + 6] = J_obs[k][:, 0:6] * fc[c]
        J[2 * k:2 * k + 2, 6 * nc + 10 * g:6 * nc + 10 * g + 10] = J_obs[k][:, 6:16] * fi[g]
        J[2 * k:2 * k + 2, 6 * nc + 10 * ng + 4 * q:6 * nc + 10 * ng + 4 * q + 4] = J_obs[k][:, 16:20] * fp[q]
    return J


FOUNTAIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fountain11_ir.npz")


def fountain_problem(intrinsics_to_optimize=_abi.INTR_NONE):
    """The reference's fountain-11 reconstruction as a Problem (shared PINHOLE intrinsics; constant by default, as in
    the run that produced it: the stored intrinsics equal the ground-truth calibration exactly)."""
    g = np.load(FOUNTAIN)
    n = len(g["names"])
    mask = _abi.constant_intrinsics_mask(_abi.MODEL_PINHOLE, intrinsics_to_optimize)
    p = _abi.Problem(g["ext"], np.zeros(n, np.uint8), np.zeros(n, np.int32), [_abi.MODEL_PINHOLE], g["intr"], [mask], g["pt"],
                     np.zeros(len(g["pt"]), np.uint8), g["obs_cam"], g["obs_pt"], g["obs_xy"])
    return p, g


def umeyama_align(src, dst):
    """Similarity transform (scale, rotation, translation) minimising |s R src + t - dst| (Umeyama 1991); what
    AlignReconstructions (transformation/align_reconstructions.cc:97-130) applies to camera positions."""
    src = np.asarray(src, float); dst = np.asarray(dst, float)
    mu_s, mu_d = src.mean(0), dst.mean(0)
    xs, xd = src - mu_s, dst - mu_d
    U, S, Vt = np.linalg.svd(xd.T @ xs / len(src))
    D = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        D[2, 2] = -1
    R = U @ D @ Vt
    scale = np.trace(np.diag(S) @ D) / (xs ** 2).sum() * len(src)
    t = mu_d - scale * R @ mu_s
    return (scale * (R @ src.T)).T + t, scale
