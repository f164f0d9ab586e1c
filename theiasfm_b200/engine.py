"""ctypes binding of the C-ABI (include/theia_ba_b200.h) -> theiasfm_b200/libtheia_ba_b200.so.

There is NO CPU fallback: if the CUDA library is missing, or no CUDA device is visible, construction
of an ``Engine`` raises.  The product path never touches ``oracle/``.
"""
import ctypes as C
import os

import numpy as np

from . import _abi

_HERE = os.path.dirname(os.path.abspath(__file__))
# THEIA_BA_B200_LIB overrides where the C-ABI library is loaded from (an out-of-tree install; the test suite's emulation build,
# which spawned rank processes must find too).  Whatever it names must export the full ABI: there is no CPU fallback.
LIB_PATH = os.environ.get("THEIA_BA_B200_LIB") or os.path.join(_HERE, "libtheia_ba_b200.so")
_LIB = None

# every symbol include/theia_ba_b200.h declares
EXPORTED_SYMBOLS = [
    "tba_options_init", "tba_device_count", "tba_create", "tba_destroy", "tba_nccl_unique_id", "tba_last_error",
    "tba_solve", "tba_upload", "tba_minimize", "tba_download", "tba_shard_points", "tba_debug_linearize", "tba_debug_linearize_raw",
    "tba_debug_stream_launch", "tba_debug_intr_cols",
    "tba_debug_prepare_linear_system", "tba_debug_schur_matvec", "tba_debug_solve_linear_system",
    "tba_debug_evaluate_step", "tba_debug_read", "tba_reset_parameters", "tba_set_max_iterations", "tba_set_profiling", "tba_get_profile", "tba_get_profile_stages", "tba_solve_multi", "tba_debug_pack", "tba_filter_tracks", "tba_adjust_tracks", "tba_adjust_views", "tba_estimate_tracks", "tba_two_view_ba_batch", "tba_two_view_ba_batch_multi",
]


class EngineError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("tba error %d: %s" % (code, message))
        self.code = code


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(make -C theiasfm_b200/csrc). There is no CPU fallback." % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        dp = C.POINTER(C.c_double)
        L.tba_options_init.argtypes = [C.POINTER(_abi.tba_options)]
        L.tba_device_count.restype = C.c_int
        L.tba_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]
        L.tba_destroy.argtypes = [C.c_void_p]
        L.tba_nccl_unique_id.argtypes = [C.c_void_p]
        L.tba_last_error.restype = C.c_char_p
        L.tba_last_error.argtypes = [C.c_void_p]
        L.tba_solve.argtypes = [C.c_void_p, C.POINTER(_abi.tba_options), C.POINTER(_abi.tba_problem), C.POINTER(_abi.tba_summary)]
        L.tba_upload.argtypes = [C.c_void_p, C.POINTER(_abi.tba_options), C.POINTER(_abi.tba_problem)]
        L.tba_minimize.argtypes = [C.c_void_p, C.POINTER(_abi.tba_summary)]
        L.tba_download.argtypes = [C.c_void_p, C.POINTER(_abi.tba_problem)]
        L.tba_shard_points.argtypes = [C.POINTER(C.c_int32), C.c_int32, C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        L.tba_debug_linearize.argtypes = [C.c_void_p, dp]
        L.tba_debug_linearize_raw.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int64), dp, dp, dp, dp, dp]
        L.tba_debug_stream_launch.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        L.tba_debug_intr_cols.argtypes = [C.c_void_p, C.POINTER(C.c_int64), dp]
        L.tba_debug_prepare_linear_system.argtypes = [C.c_void_p, C.c_double]
        L.tba_debug_schur_matvec.argtypes = [C.c_void_p, dp, dp, dp, dp]
        L.tba_debug_solve_linear_system.argtypes = [C.c_void_p, C.POINTER(C.c_int32), dp]
        L.tba_debug_evaluate_step.argtypes = [C.c_void_p, dp]
        L.tba_debug_read.argtypes = [C.c_void_p, C.c_int, dp, C.c_int64]
        L.tba_abi_sizes.argtypes = [C.POINTER(C.c_int32)]
        L.tba_solve_multi.argtypes = [C.POINTER(_abi.tba_options), C.POINTER(_abi.tba_problem), C.POINTER(_abi.tba_summary), C.c_int]
        L.tba_debug_pack.restype = C.c_int
        L.tba_adjust_tracks.argtypes = [C.c_void_p, C.POINTER(_abi.tba_options), C.POINTER(C.c_uint8), dp, dp, C.POINTER(C.c_int32)]
        L.tba_adjust_views.argtypes = [C.c_void_p, C.POINTER(_abi.tba_options), C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_uint8), dp, dp,
                                       C.POINTER(C.c_int32)]
        L.tba_estimate_tracks.argtypes = [C.c_void_p, C.POINTER(_abi.tba_options), C.c_double, C.c_double, C.c_int32, C.POINTER(C.c_uint8), C.POINTER(C.c_int32)]
        L.tba_two_view_ba_batch_multi.argtypes = [C.POINTER(_abi.tba_two_view_batch), C.c_int, C.POINTER(C.c_uint8), dp, dp, C.POINTER(C.c_int32)]
        L.tba_two_view_ba_batch.argtypes = [C.c_void_p, C.POINTER(_abi.tba_two_view_batch), C.POINTER(C.c_uint8), dp, dp, C.POINTER(C.c_int32)]
        L.tba_filter_tracks.argtypes = [C.c_void_p, C.c_double, C.c_double, C.POINTER(C.c_uint8), dp, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        L.tba_reset_parameters.argtypes = [C.c_void_p, C.POINTER(_abi.tba_problem)]
        L.tba_set_max_iterations.argtypes = [C.c_void_p, C.c_int32]
        L.tba_set_profiling.argtypes = [C.c_void_p, C.c_int]
        L.tba_get_profile.argtypes = [C.c_void_p, dp]
        L.tba_get_profile_stages.argtypes = [C.c_void_p, dp]
        _LIB = L
    return _LIB


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def default_options(**kw):
    """theia::BundleAdjustmentOptions defaults (bundle_adjustment.h:78-122) + Ceres' defaults."""
    o = _abi.tba_options()
    lib().tba_options_init(C.byref(o))
    for k, v in kw.items():
        if not hasattr(o, k):
            raise AttributeError(k)
        setattr(o, k, v)
    return o


def device_count():
    return lib().tba_device_count()


def nccl_unique_id():
    buf = C.create_string_buffer(128)
    rc = lib().tba_nccl_unique_id(buf)
    if rc != 0:
        raise EngineError(rc, "ncclGetUniqueId failed")
    return buf.raw


def shard_points(pt_num_obs, world_size, rank):
    a = np.ascontiguousarray(pt_num_obs, dtype=np.int32)
    b, e = C.c_int32(), C.c_int32()
    lib().tba_shard_points(a.ctypes.data_as(C.POINTER(C.c_int32)), len(a), world_size, rank, C.byref(b), C.byref(e))
    return b.value, e.value


class Summary:
    def __init__(self, s, iters):
        for f, _ in _abi.tba_summary._fields_:
            if f not in ("iterations", "message"):
                setattr(self, f, getattr(s, f))
        self.message = s.message.decode(errors="replace")
        n = min(s.num_iterations, len(iters))
        self.iterations = [{f: getattr(iters[i], f) for f, _ in _abi.tba_iteration._fields_} for i in range(n)]

    @property
    def costs(self):
        return np.array([it["cost"] for it in self.iterations])


def debug_pack(problem):
    """tba_debug_pack: the host-side tile packing (no GPU needed). Returns a dict of numpy arrays."""
    cap = (problem.n_obs // 200 + problem.n_pt // 8 + 8) * 256 + problem.n_obs * 2
    sizes = np.zeros(6, np.int64)
    out = dict(slot_cam=np.zeros(cap, np.int32), slot_pt=np.zeros(cap, np.int32), slot_run=np.zeros(cap, np.int16),
               slot_flags=np.zeros(cap, np.uint8), xy=np.zeros(cap * 2), slot_orig=np.zeros(cap, np.int64),
               pk2caller=np.zeros(max(problem.n_pt, 1), np.int32), tile_pt_begin=np.zeros(cap // 256 + 2, np.int32),
               tile_nruns=np.zeros(cap // 256 + 2, np.int32), tile_flags=np.zeros(cap // 256 + 2, np.uint8),
               mask=np.zeros(problem.n_cam * 6 + problem.n_group * 10))
    st = problem.as_struct()
    P = C.POINTER
    rc = lib().tba_debug_pack(C.byref(st), cap, sizes.ctypes.data_as(P(C.c_int64)), out["slot_cam"].ctypes.data_as(P(C.c_int32)),
                              out["slot_pt"].ctypes.data_as(P(C.c_int32)), out["slot_run"].ctypes.data_as(P(C.c_int16)),
                              out["slot_flags"].ctypes.data_as(P(C.c_uint8)), _dp(out["xy"]), out["slot_orig"].ctypes.data_as(P(C.c_int64)),
                              out["pk2caller"].ctypes.data_as(P(C.c_int32)), out["tile_pt_begin"].ctypes.data_as(P(C.c_int32)),
                              out["tile_nruns"].ctypes.data_as(P(C.c_int32)), out["tile_flags"].ctypes.data_as(P(C.c_uint8)), _dp(out["mask"]))
    n_tiles, n_slots, npk, n_long, ni, imask = (int(v) for v in sizes)
    out.update(rc=rc, n_tiles=n_tiles, n_slots=n_slots, n_packed_points=npk, n_long_points=n_long, NI=ni, imask=imask)
    if rc == 0:
        for k in ("slot_cam", "slot_pt", "slot_run", "slot_flags", "slot_orig"):
            out[k] = out[k][:n_slots]
        out["xy"] = out["xy"][:n_slots * 2]
        out["pk2caller"] = out["pk2caller"][:npk]
        out["tile_pt_begin"] = out["tile_pt_begin"][:n_tiles + 1]
        out["tile_nruns"] = out["tile_nruns"][:n_tiles]
        out["tile_flags"] = out["tile_flags"][:n_tiles]
    return out


def two_view_ba_batch_multi(batch, n_devices=0):
    """tba_two_view_ba_batch_multi: the batch sharded by pairs over n_devices GPUs (0 = all); updates the batch in place."""
    n = max(batch.n_pairs, 1)
    term = np.zeros(n, np.uint8); ic = np.zeros(n); fc = np.zeros(n); it = np.zeros(n, np.int32)
    st = batch.as_struct()
    rc = lib().tba_two_view_ba_batch_multi(C.byref(st), n_devices, term.ctypes.data_as(C.POINTER(C.c_uint8)), _dp(ic), _dp(fc),
                                           it.ctypes.data_as(C.POINTER(C.c_int32)))
    if rc != 0:
        raise EngineError(rc, "tba_two_view_ba_batch_multi failed")
    n = batch.n_pairs
    return term[:n], ic[:n], fc[:n], it[:n]


def solve_multi(problem, options=None, n_devices=0, max_iterations_logged=2048):
    """tba_solve_multi: single-process multi-GPU solve (one host thread per device inside the library)."""
    options = options or default_options()
    iters = (_abi.tba_iteration * max_iterations_logged)()
    s = _abi.tba_summary()
    s.iterations = C.cast(iters, C.POINTER(_abi.tba_iteration))
    s.iterations_capacity = max_iterations_logged
    st = problem.as_struct()
    rc = lib().tba_solve_multi(C.byref(options), C.byref(st), C.byref(s), n_devices)
    out = Summary(s, iters)
    out.rc = rc
    return out


class Engine:
    """One GPU's engine context (tba_create / tba_destroy)."""

    def __init__(self, device=0, rank=0, world_size=1, nccl_id=None, max_iterations_logged=2048):
        L = lib()
        if L.tba_device_count() <= 0:
            raise EngineError(_abi.ERR_NO_DEVICE, "no CUDA device visible; the engine has no CPU fallback")
        h = C.c_void_p()
        idbuf = C.create_string_buffer(nccl_id, 128) if nccl_id is not None else None
        rc = L.tba_create(device, rank, world_size, idbuf, C.byref(h))
        if rc != 0:
            raise EngineError(rc, "tba_create failed")
        self._h = h
        self.rank, self.world_size = rank, world_size
        self._iters = (_abi.tba_iteration * max_iterations_logged)()
        self._problem = None

    def close(self):
        if getattr(self, "_h", None):
            lib().tba_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise EngineError(rc, lib().tba_last_error(self._h).decode(errors="replace"))

    def _new_summary(self):
        s = _abi.tba_summary()
        s.iterations = C.cast(self._iters, C.POINTER(_abi.tba_iteration))
        s.iterations_capacity = len(self._iters)
        return s

    # ---- whole solve: host buffers in, host buffers out (the drop-in call)
    def solve(self, problem, options=None):
        options = options or default_options()
        s = self._new_summary()
        st = problem.as_struct()
        self._problem = problem
        rc = lib().tba_solve(self._h, C.byref(options), C.byref(st), C.byref(s))
        out = Summary(s, self._iters)
        out.rc = rc
        if rc != 0:
            out.message = lib().tba_last_error(self._h).decode(errors="replace")
        return out

    # ---- split phase
    def upload(self, problem, options=None):
        options = options or default_options()
        self._problem = problem
        self._st = problem.as_struct()
        self._check(lib().tba_upload(self._h, C.byref(options), C.byref(self._st)))

    def minimize(self):
        s = self._new_summary()
        self._check(lib().tba_minimize(self._h, C.byref(s)))
        out = Summary(s, self._iters)
        out.rc = 0  # a failure raised above; same attribute as the summary of solve()
        return out

    def download(self, problem=None):
        problem = problem or self._problem
        st = problem.as_struct()
        self._check(lib().tba_download(self._h, C.byref(st)))

    def filter_tracks(self, max_inlier_reprojection_error, min_triangulation_angle_degrees):
        """tba_filter_tracks on the device-resident problem: (status [n_pt] uint8, mean_sq_error [n_pt], n_bad, n_insufficient)."""
        n = self._problem.n_pt
        status = np.zeros(max(n, 1), np.uint8); mean = np.zeros(max(n, 1))
        nb, ni = C.c_int32(), C.c_int32()
        self._check(lib().tba_filter_tracks(self._h, max_inlier_reprojection_error, min_triangulation_angle_degrees,
                                            status.ctypes.data_as(C.POINTER(C.c_uint8)), _dp(mean), C.byref(nb), C.byref(ni)))
        return status[:n], mean[:n], nb.value, ni.value

    def adjust_tracks(self, options):
        """tba_adjust_tracks (batched BundleAdjustTrack) on the device-resident problem; call download() for the points.
        Returns (status [n_pt] uint8, initial_cost, final_cost, n_failed)."""
        n = max(self._problem.n_pt, 1)
        status = np.zeros(n, np.uint8); ic = np.zeros(n); fc = np.zeros(n); nf = C.c_int32()
        self._check(lib().tba_adjust_tracks(self._h, C.byref(options), status.ctypes.data_as(C.POINTER(C.c_uint8)), _dp(ic), _dp(fc), C.byref(nf)))
        n = self._problem.n_pt
        return status[:n], ic[:n], fc[:n], nf.value

    def adjust_views(self, options, views):
        """tba_adjust_views (batched BundleAdjustView) on the device-resident problem for the cameras `views`; call download() for
        the refined extrinsics and intrinsics.  Returns (status [n] uint8, initial_cost [n], final_cost [n], iterations [n] int32)."""
        v = np.ascontiguousarray(views, dtype=np.int32).reshape(-1)
        n = len(v)
        status = np.zeros(max(n, 1), np.uint8); ic = np.zeros(max(n, 1)); fc = np.zeros(max(n, 1)); it = np.zeros(max(n, 1), np.int32)
        self._check(lib().tba_adjust_views(self._h, C.byref(options), v.ctypes.data_as(C.POINTER(C.c_int32)), n,
                                           status.ctypes.data_as(C.POINTER(C.c_uint8)), _dp(ic), _dp(fc), it.ctypes.data_as(C.POINTER(C.c_int32))))
        return status[:n], ic[:n], fc[:n], it[:n]

    def estimate_tracks(self, options, max_reprojection_error_pixels=5.0, min_triangulation_angle_degrees=3.0, bundle_adjustment=True):
        """tba_estimate_tracks (batched TrackEstimator::EstimateTrack); call download() for the points. Returns (status, counts[5])."""
        status = np.zeros(max(self._problem.n_pt, 1), np.uint8); counts = np.zeros(5, np.int32)
        self._check(lib().tba_estimate_tracks(self._h, C.byref(options), max_reprojection_error_pixels, min_triangulation_angle_degrees,
                                              int(bundle_adjustment), status.ctypes.data_as(C.POINTER(C.c_uint8)),
                                              counts.ctypes.data_as(C.POINTER(C.c_int32))))
        return status[:self._problem.n_pt], counts

    def two_view_ba_batch(self, batch):
        """tba_two_view_ba_batch (batched BundleAdjustTwoViews): updates batch.ext2 / intr1 / intr2 / points in place.
        Returns (termination [n_pairs] uint8, initial_cost, final_cost, iterations)."""
        n = max(batch.n_pairs, 1)
        term = np.zeros(n, np.uint8); ic = np.zeros(n); fc = np.zeros(n); it = np.zeros(n, np.int32)
        st = batch.as_struct()
        self._check(lib().tba_two_view_ba_batch(self._h, C.byref(st), term.ctypes.data_as(C.POINTER(C.c_uint8)), _dp(ic), _dp(fc),
                                                it.ctypes.data_as(C.POINTER(C.c_int32))))
        n = batch.n_pairs
        return term[:n], ic[:n], fc[:n], it[:n]

    def reset_parameters(self, problem):
        st = problem.as_struct()
        self._check(lib().tba_reset_parameters(self._h, C.byref(st)))

    def set_max_iterations(self, n):
        self._check(lib().tba_set_max_iterations(self._h, int(n)))

    def set_profiling(self, enable=True):
        self._check(lib().tba_set_profiling(self._h, int(enable)))

    def profile(self):
        out = np.zeros(8)
        self._check(lib().tba_get_profile(self._h, _dp(out)))
        return dict(matvec_ms=out[0], matvec_launches=int(out[1]), linearize_ms=out[2], linearize_launches=int(out[3]),
                    slots=int(out[4]), observations=int(out[5]), points=int(out[6]), doubles_per_obs=int(out[7]))

    STAGES = ("matvec", "linearize", "precond_ext", "precond_intr", "rhs", "backsub", "candidate_cost", "prepare_fused")

    def profile_stages(self):
        """Per-stage device time of the profiled run: {stage: {"ms": total, "launches": n}} (tba_get_profile_stages)."""
        out = np.zeros(16)
        self._check(lib().tba_get_profile_stages(self._h, _dp(out)))
        return {k: {"ms": float(out[2 * i]), "launches": int(out[2 * i + 1])} for i, k in enumerate(self.STAGES)}

    # ---- stage hooks (kernel-level parity tests)
    def linearize(self):
        c = C.c_double()
        rc = lib().tba_debug_linearize(self._h, C.byref(c))
        return rc == 0, c.value

    def linearize_raw(self, tile_kernel=False):
        """tba_debug_linearize_raw: one linearisation; the raw device buffers J [slices, NJ, 32], res [slices, 2, 32], Hpp [n_pt, 10],
        gp [n_pt, 4] (packed points) and lin = gradient | squared column norms | cost, fixed cost, failed evaluations.
        tile_kernel: the tile-per-CTA kernel over every tile instead of the streaming kernel over the normal tiles."""
        sizes = np.zeros(4, np.int64)
        self._check(lib().tba_debug_linearize_raw(self._h, int(tile_kernel), sizes.ctypes.data_as(C.POINTER(C.c_int64)), None, None, None, None, None))
        n_slots, nj, n_pt, ncs = (int(v) for v in sizes)
        J, res = np.zeros((n_slots // 32, nj, 32)), np.zeros((n_slots // 32, 2, 32))
        Hpp, gp, lin = np.zeros((n_pt, 10)), np.zeros((n_pt, 4)), np.zeros(2 * ncs + 3)
        self._check(lib().tba_debug_linearize_raw(self._h, int(tile_kernel), sizes.ctypes.data_as(C.POINTER(C.c_int64)),
                                                  _dp(J), _dp(res), _dp(Hpp), _dp(gp), _dp(lin)))
        return dict(J=J, res=res, Hpp=Hpp, gp=gp, g=lin[:ncs], cn=lin[ncs:2 * ncs], cost=lin[2 * ncs], fixed=lin[2 * ncs + 1],
                    failed=lin[2 * ncs + 2])

    def intr_cols_raw(self):
        """tba_debug_intr_cols: J_i [slices, 2 NI, 32] of the last linearisation as the passes over J see it (rebuilt from the stored
        normalised image point in the compact layout), in the order of linearize_raw()["J"][:, 14:] in the full layout."""
        sizes = np.zeros(2, np.int64)
        self._check(lib().tba_debug_intr_cols(self._h, sizes.ctypes.data_as(C.POINTER(C.c_int64)), None))
        n_slots, ni = (int(v) for v in sizes)
        Ji = np.zeros((n_slots // 32, 2 * ni, 32))
        self._check(lib().tba_debug_intr_cols(self._h, sizes.ctypes.data_as(C.POINTER(C.c_int64)), _dp(Ji)))
        return Ji

    STREAM_KERNELS = ("linearize", "prepare", "matvec", "rhs_backsub")

    def stream_launch(self):
        """tba_debug_stream_launch: the launch geometry of the persistent warp-slice kernels over the uploaded normal tiles.
        {n_sm, n_slices, imask, has_ext_models, and per kernel in STREAM_KERNELS: {grid, NW, NS}}; k_linearize_stream,
        k_prepare_stream, k_schur_stream MODE 0 and MODE 1 / 2.  Warp gw of GW = grid * NW owns [n_slices*gw/GW, n_slices*(gw+1)/GW)."""
        out = np.zeros(16, np.int32)
        self._check(lib().tba_debug_stream_launch(self._h, out.ctypes.data_as(C.POINTER(C.c_int32))))
        d = dict(n_sm=int(out[0]), n_slices=int(out[1]), imask=int(out[2]), has_ext_models=bool(out[3]))
        for k, name in enumerate(self.STREAM_KERNELS):
            d[name] = dict(grid=int(out[4 + 3 * k]), NW=int(out[5 + 3 * k]), NS=int(out[6 + 3 * k]))
        return d

    def prepare_linear_system(self, radius):
        return lib().tba_debug_prepare_linear_system(self._h, radius) == 0

    def schur_matvec(self, x_cam, x_intr):
        x_cam = np.ascontiguousarray(x_cam, np.float64); x_intr = np.ascontiguousarray(x_intr, np.float64)
        y_cam = np.zeros_like(x_cam); y_intr = np.zeros_like(x_intr)
        self._check(lib().tba_debug_schur_matvec(self._h, _dp(x_cam), _dp(x_intr), _dp(y_cam), _dp(y_intr)))
        return y_cam, y_intr

    def solve_linear_system(self):
        it, m = C.c_int32(), C.c_double()
        rc = lib().tba_debug_solve_linear_system(self._h, C.byref(it), C.byref(m))
        return rc == 0, it.value, m.value

    def evaluate_step(self):
        c = C.c_double()
        rc = lib().tba_debug_evaluate_step(self._h, C.byref(c))
        return rc == 0, c.value

    def read(self, which):
        p = self._problem
        n = {_abi.VEC_GRADIENT_CAM: p.n_cam * 6, _abi.VEC_GRADIENT_INTR: p.n_group * 10, _abi.VEC_GRADIENT_PT: p.n_pt * 4,
             _abi.VEC_COLNORM2_CAM: p.n_cam * 6, _abi.VEC_COLNORM2_INTR: p.n_group * 10, _abi.VEC_COLNORM2_PT: p.n_pt * 4,
             _abi.VEC_RESIDUALS: p.n_obs * 2, _abi.VEC_SCHUR_RHS_CAM: p.n_cam * 6, _abi.VEC_SCHUR_RHS_INTR: p.n_group * 10,
             _abi.VEC_PRECOND_CAM: p.n_cam * 36, _abi.VEC_PRECOND_INTR: p.n_group * 100, _abi.VEC_STEP_CAM: p.n_cam * 6,
             _abi.VEC_STEP_INTR: p.n_group * 10, _abi.VEC_STEP_PT: p.n_pt * 4}[which]
        out = np.zeros(n)
        self._check(lib().tba_debug_read(self._h, which, _dp(out), n))
        return out
