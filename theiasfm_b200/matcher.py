"""ctypes binding of include/theia_matcher_b200.h -> theiasfm_b200/libtheia_matcher_b200.so (secondary path, SURVEY row a16).
No CPU fallback: tbm_match_all fails with -5 when no GPU is visible."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtheia_matcher_b200.so")
_LIB = None
EXPORTED_SYMBOLS = ["tbm_options_init", "tbm_match_all", "tbm_debug_postprocess", "tbm_debug_last_timing", "tbm_debug_exact_top2",
                    "tbm_debug_nn2"]


class tbm_match(C.Structure):
    _fields_ = [("feature1_ind", C.c_int32), ("feature2_ind", C.c_int32), ("distance", C.c_float)]


class tbm_options(C.Structure):
    _fields_ = [("keep_only_symmetric_matches", C.c_int32), ("use_lowes_ratio", C.c_int32), ("lowes_ratio", C.c_float),
                ("min_num_feature_matches", C.c_int32)]


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("%s is missing: build it with make -C theiasfm_b200/csrc (no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        L.tbm_options_init.argtypes = [C.POINTER(tbm_options)]
        L.tbm_match_all.argtypes = [C.c_int, fp, C.POINTER(C.c_int64), C.c_int32, C.c_int32, ip, C.c_int64, C.POINTER(tbm_options),
                                    C.POINTER(tbm_match), C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_uint8)]
        L.tbm_debug_postprocess.argtypes = [ip, fp, fp, C.c_int32, C.c_int, ip, fp, fp, C.c_int32, C.c_int, C.POINTER(tbm_options),
                                            C.POINTER(tbm_match), ip]
        L.tbm_debug_last_timing.argtypes = [C.POINTER(C.c_double)]
        L.tbm_debug_last_timing.restype = None
        L.tbm_debug_exact_top2.argtypes = [C.c_int, fp, C.c_int64, ip, ip, ip, ip, C.c_int64, ip, fp, fp]
        L.tbm_debug_nn2.argtypes = [C.c_int, fp, C.POINTER(C.c_int64), C.c_int32, C.c_int32, ip, C.c_int64, C.c_int, ip, fp, fp,
                                    C.POINTER(C.c_uint8)]
        _LIB = L
    return _LIB


def last_timing():
    """{gemm_ms, exact_ms, h2d_ms} of the last match_all on the tensor-core path (CUDA events)."""
    out = (C.c_double * 4)()
    lib().tbm_debug_last_timing(out)
    return {"gemm_ms": out[0], "exact_ms": out[1], "h2d_ms": out[2], "exhaustive_queries": out[3]}


def exact_top2(descriptors, q_row, b_row0, b_rows, cand, device=0):
    """tbm_debug_exact_top2: the exact re-evaluation kernel of the tensor-core path on hand-made candidate lists [n_q, 16]."""
    d = np.ascontiguousarray(descriptors, np.float32)
    q = np.ascontiguousarray(q_row, np.int32); b0 = np.ascontiguousarray(b_row0, np.int32); bn = np.ascontiguousarray(b_rows, np.int32)
    cd = np.ascontiguousarray(cand, np.int32)
    n = len(q)
    bj = np.zeros(n, np.int32); bd = np.zeros(n, np.float32); sd = np.zeros(n, np.float32)
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    rc = lib().tbm_debug_exact_top2(device, d.ctypes.data_as(fp), len(d), q.ctypes.data_as(ip), b0.ctypes.data_as(ip), bn.ctypes.data_as(ip),
                                    cd.ctypes.data_as(ip), n, bj.ctypes.data_as(ip), bd.ctypes.data_as(fp), sd.ctypes.data_as(fp))
    return rc, bj, bd, sd


def _pack(descriptor_sets, pairs):
    dim = descriptor_sets[0].shape[1]
    off = np.zeros(len(descriptor_sets) + 1, np.int64)
    off[1:] = np.cumsum([len(d) for d in descriptor_sets])
    desc = np.ascontiguousarray(np.concatenate(descriptor_sets, axis=0), np.float32) if off[-1] else np.zeros((0, dim), np.float32)
    pr = np.ascontiguousarray(np.array(pairs, np.int32).reshape(-1, 2))
    return dim, off, desc, pr


def nn2(descriptor_sets, pairs, symmetric=True, device=0):
    """tbm_debug_nn2: the per-query nearest / second-nearest results of tbm_match_all's search stage.
    Returns (rc, [per pair: dict(fwd=(best_j, best_d, second_d, exhaustive), rev=(...) or None)])."""
    dim, off, desc, pr = _pack(descriptor_sets, pairs)
    sizes = np.diff(off)
    nq = int(sum(sizes[a] + (sizes[b] if symmetric else 0) for a, b in pr))
    bj = np.zeros(max(nq, 1), np.int32); bd = np.zeros(max(nq, 1), np.float32); sd = np.zeros(max(nq, 1), np.float32)
    ex = np.zeros(max(nq, 1), np.uint8)
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    rc = lib().tbm_debug_nn2(device, desc.ctypes.data_as(fp), off.ctypes.data_as(C.POINTER(C.c_int64)), len(descriptor_sets), dim,
                             pr.ctypes.data_as(ip), len(pr), int(bool(symmetric)), bj.ctypes.data_as(ip), bd.ctypes.data_as(fp),
                             sd.ctypes.data_as(fp), ex.ctypes.data_as(C.POINTER(C.c_uint8)))
    res, q = [], 0
    for a, b in pr:
        part = {}
        for key, n in (("fwd", sizes[a]), ("rev", sizes[b] if symmetric else None)):
            if n is None:
                part[key] = None
                continue
            n = int(n)
            part[key] = (bj[q:q + n], bd[q:q + n], sd[q:q + n], ex[q:q + n].astype(bool))
            q += n
        res.append(part)
    return rc, res


def default_options(**kw):
    o = tbm_options()
    lib().tbm_options_init(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def match_all(descriptor_sets, pairs, options=None, device=0):
    """descriptor_sets: list of [n_i, dim] float32 arrays; pairs: [(i, j), ...].
    Returns (rc, [list of (f1, f2, dist) per pair], [ok per pair])."""
    options = options or default_options()
    dim, off, desc, pr = _pack(descriptor_sets, pairs)
    cap = int(sum(len(descriptor_sets[i]) for i, _ in pairs)) + 1
    out = (tbm_match * cap)()
    moff = np.zeros(len(pr) + 1, np.int64)
    ok = np.zeros(max(len(pr), 1), np.uint8)
    rc = lib().tbm_match_all(device, desc.ctypes.data_as(C.POINTER(C.c_float)), off.ctypes.data_as(C.POINTER(C.c_int64)), len(descriptor_sets),
                             dim, pr.ctypes.data_as(C.POINTER(C.c_int32)), len(pr), C.byref(options), out, cap,
                             moff.ctypes.data_as(C.POINTER(C.c_int64)), ok.ctypes.data_as(C.POINTER(C.c_uint8)))
    res = []
    if rc == 0:
        for p in range(len(pr)):
            res.append([(out[k].feature1_ind, out[k].feature2_ind, out[k].distance) for k in range(int(moff[p]), int(moff[p + 1]))])
    return rc, res, [bool(v) for v in ok[:len(pr)]]
