"""The matcher on the GPU against plain float references at the inputs where its tensor-core candidate pass can go wrong:
  * the adversarial classes of tests/matcher_cases.py (zero rows, disjoint supports, near-ties below TF32 resolution, signed
    descriptors with norm disparity, integer-valued and scaled descriptors) through tbm_debug_nn2 -- the raw nearest / second-nearest
    results, bit for bit against the reference's float arithmetic -- and through tbm_match_all against the CPU oracle, on both paths;
  * image sizes around the 64-row candidate tile and the 128-row query block, with the smallest image last (TMA out-of-bounds fill);
  * the host loops at scale: more than 4 M queries (two chunks), more than 4096 pairs and 8192 query segments, empty images;
  * the capacity contract of tbm_match_all;
  * the CUDA-core kernel k_nn2 at dimensions other than 128, including the > 48 KB shared-memory configuration.
Under --emulate-engine only the CUDA-core path exists (every dim) and the scale cases are skipped."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import matcher_cases as mc
from test_matcher_host import _nn2_float32
from theiasfm_b200 import matcher

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_ORACLE = []


def _emulated():
    return "_emu" in os.path.basename(matcher.LIB_PATH)


def _paths():
    return ("exact",) if _emulated() else ("tc", "exact")


def _set_path(monkeypatch, path):
    if path == "exact":
        monkeypatch.setenv("TBM_PATH", "exact")
    else:
        monkeypatch.delenv("TBM_PATH", raising=False)


def _oracle_match(d1, d2, **kw):
    """oracle/matcher_oracle.c's MatchImagePair (built once per session)"""
    if not _ORACLE:
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "libmatcher_oracle.so"], stdout=subprocess.DEVNULL)
        _ORACLE.append(C.CDLL(os.path.join(ROOT, "oracle", "libmatcher_oracle.so")))
    d1 = np.ascontiguousarray(d1, np.float32); d2 = np.ascontiguousarray(d2, np.float32)
    o = matcher.default_options(**kw)
    out = (matcher.tbm_match * max(len(d1), 1))(); n = C.c_int()
    fp = C.POINTER(C.c_float)
    ok = _ORACLE[0].matcher_match_image_pair(d1.ctypes.data_as(fp), len(d1), d2.ctypes.data_as(fp), len(d2), d1.shape[1], C.byref(o), out,
                                              C.byref(n))
    return bool(ok), [(out[i].feature1_ind, out[i].feature2_ind, out[i].distance) for i in range(n.value)]


def _expected_nn2(A, B):
    if len(B) == 0:
        return np.full(len(A), -1, np.int32), np.zeros(len(A), np.float32), np.zeros(len(A), np.float32)
    return _nn2_float32(A, B)


def _check_nn2(sets, pairs, tag):
    """tbm_debug_nn2 (symmetric) against the reference's float arithmetic, bit for bit; returns the exhaustively scanned queries"""
    rc, res = matcher.nn2(sets, pairs, symmetric=True)
    assert rc == 0, (tag, rc)
    n_exh = 0
    for (a, b), r in zip(pairs, res):
        for key, (Q, Cd) in (("fwd", (sets[a], sets[b])), ("rev", (sets[b], sets[a]))):
            bj, bd, sd, ex = r[key]
            ej, ed, es = _expected_nn2(Q, Cd)
            n_exh += int(ex.sum())
            bad = np.flatnonzero((bj != ej) | (bd.view(np.uint32) != ed.view(np.uint32)) | (sd.view(np.uint32) != es.view(np.uint32)))
            assert len(bad) == 0, (tag, (a, b), key, bad[:8], bj[bad[:4]], ej[bad[:4]], bd[bad[:4]], ed[bad[:4]], sd[bad[:4]], es[bad[:4]],
                                   "exhaustive", int(ex.sum()))
    return n_exh


OPTION_SETS = (dict(), dict(use_lowes_ratio=0, min_num_feature_matches=0), dict(lowes_ratio=1.0, min_num_feature_matches=0))


def _check_match_all(sets, pairs, tag, option_sets=OPTION_SETS):
    for kw in option_sets:
        rc, res, ok = matcher.match_all(sets, pairs, matcher.default_options(**kw))
        assert rc == 0, (tag, kw, rc)
        for p, (a, b) in enumerate(pairs):
            ok_o, exp = _oracle_match(sets[a], sets[b], **kw)
            assert ok[p] == ok_o and res[p] == exp, (tag, kw, (a, b), len(res[p]), len(exp))


@pytest.mark.parametrize("cls", sorted(mc.CLASSES))
def test_adversarial_class_equals_the_reference(cls, monkeypatch):
    """every case of the class: raw top-2 of both directions bit for bit (tbm_debug_nn2), then the match lists and pair flags of
    tbm_match_all against the oracle -- default options, no ratio test, and ratio 1.0 (best strictly below second) -- on both paths"""
    exhaustive = {}
    for path in _paths():
        _set_path(monkeypatch, path)
        for name, sets, pairs in mc.CLASSES[cls]():
            exhaustive[(path, name)] = _check_nn2(sets, pairs, (path, name))
            _check_match_all(sets, pairs, (path, name, "exhaustive_queries", exhaustive))
    if "tc" in _paths():
        assert all(v == 0 for (p, _), v in exhaustive.items() if p == "exact")


@pytest.mark.skipif(_emulated(), reason="the tensor-core path does not exist in the emulation build")
def test_tf32_operands_are_truncated(monkeypatch):
    """the margin of k_nn_candidates for non-negative descriptors assumes that wgmma .tf32 truncates its fp32 operands (a score is
    never under-estimated by more than the fp32 accumulation error).  The probe of matcher_cases.truncation_probe keeps a 2-entry
    candidate list under truncation and overflows to the exhaustive scan under round-to-nearest."""
    monkeypatch.delenv("TBM_PATH", raising=False)
    Q, Cd = mc.truncation_probe()
    rc, res = matcher.nn2([Q, Cd], [(0, 1)], symmetric=False)
    assert rc == 0
    bj, bd, sd, ex = res[0]["fwd"]
    ej, ed, es = _nn2_float32(Q, Cd)
    assert bj[0] == ej[0] == 0 and bd[0] == ed[0] and sd[0] == es[0]
    assert not ex[0], "wgmma rounds TF32 operands: the NONNEG margin of k_nn_candidates needs its rounding variant"


def test_tile_and_block_edges_equal_the_reference(monkeypatch):
    """image sizes around the 64-row candidate tile and the 128-row query block, in both roles and against themselves, the one-row
    image stored last (its TMA tile reaches past the end of the descriptor array)"""
    rng = np.random.default_rng(21)
    sizes = [2, 63, 64, 65, 127, 128, 129, 192, 256, 257, 1] if not _emulated() else [2, 63, 65, 129, 1]
    base = np.abs(rng.normal(size=(300, 128))).astype(np.float32)
    sets = []
    for n in sizes:
        s = base[rng.permutation(300)[:n]] + 0.1 * np.abs(rng.normal(size=(n, 128))).astype(np.float32)
        sets.append(np.ascontiguousarray(s / np.linalg.norm(s, axis=1, keepdims=True), np.float32))
    k = len(sizes)
    mid = sizes.index(129)
    pairs = [(i, i) for i in range(k)] + [(i, mid) for i in range(k) if i != mid] + [(mid, i) for i in range(k) if i != mid] + \
            [(k - 1, i) for i in range(k - 1)] + [(i, k - 1) for i in range(k - 1)]
    for path in _paths():
        _set_path(monkeypatch, path)
        _check_nn2(sets, pairs, (path, "sizes"))
        _check_match_all(sets, pairs, (path, "sizes"), option_sets=OPTION_SETS[:2])


def test_empty_images_equal_the_reference(monkeypatch):
    rng = np.random.default_rng(22)
    a = np.abs(rng.normal(size=(70, 128))).astype(np.float32)
    sets = [a, np.zeros((0, 128), np.float32), np.ascontiguousarray(a[::-1] + 0.01), np.zeros((0, 128), np.float32)]
    pairs = [(0, 1), (1, 0), (1, 3), (1, 1), (0, 2), (3, 2)]
    for path in _paths():
        _set_path(monkeypatch, path)
        _check_nn2(sets, pairs, (path, "empty"))
        _check_match_all(sets, pairs, (path, "empty"), option_sets=OPTION_SETS[:2])


def _raw_match_all(sets, pairs, options, cap, extra=0, sentinel=-7):
    """tbm_match_all through ctypes with host buffers (as bench.py calls it); `extra` sentinel entries behind the capacity"""
    dim, off, desc, pr = matcher._pack(sets, pairs)
    out = (matcher.tbm_match * (cap + extra + 1))()
    arr = np.frombuffer(out, dtype=np.dtype([("i", np.int32), ("j", np.int32), ("d", np.float32)]))
    arr["i"] = sentinel; arr["j"] = sentinel; arr["d"] = sentinel
    moff = np.zeros(len(pr) + 1, np.int64)
    ok = np.zeros(max(len(pr), 1), np.uint8)
    rc = matcher.lib().tbm_match_all(0, desc.ctypes.data_as(C.POINTER(C.c_float)), off.ctypes.data_as(C.POINTER(C.c_int64)), len(sets), dim,
                                     pr.ctypes.data_as(C.POINTER(C.c_int32)), len(pr), C.byref(options), out, cap,
                                     moff.ctypes.data_as(C.POINTER(C.c_int64)), ok.ctypes.data_as(C.POINTER(C.c_uint8)))
    return rc, moff, ok[:len(pr)].copy(), arr.copy()


def test_capacity_contract(monkeypatch):
    """capacity one short: -1, match_off[n_pairs] = the required capacity, nothing written past the capacity; capacity exact: the
    lists of a generous call"""
    rng = np.random.default_rng(23)
    base = np.abs(rng.normal(size=(150, 128))).astype(np.float32)
    sets = [np.ascontiguousarray(base[rng.permutation(150)[:n]] + 0.02 * np.abs(rng.normal(size=(n, 128))).astype(np.float32)) for n in (150, 120, 90)]
    pairs = [(0, 1), (1, 2), (2, 0), (0, 0)]
    opt = matcher.default_options(min_num_feature_matches=0)
    for path in _paths():
        _set_path(monkeypatch, path)
        rc, moff, ok, arr = _raw_match_all(sets, pairs, opt, 1000)
        assert rc == 0
        need = int(moff[-1])
        assert need > 100
        rc1, moff1, _, arr1 = _raw_match_all(sets, pairs, opt, need - 1, extra=8)
        assert rc1 == -1 and int(moff1[-1]) == need, (path, rc1, moff1[-1], need)
        assert np.all(arr1["i"][need - 1:] == -7) and np.all(arr1["j"][need - 1:] == -7) and np.all(arr1["d"][need - 1:] == -7)
        rc2, moff2, ok2, arr2 = _raw_match_all(sets, pairs, opt, need, extra=8)
        assert rc2 == 0 and np.array_equal(moff2, moff) and np.array_equal(ok2, ok)
        assert np.array_equal(arr2[:need], arr[:need]) and np.all(arr2["i"][need:] == -7)


@pytest.mark.parametrize("dim", [1, 3, 4, 31, 33, 64, 127, 129, 175, 176, 191, 192, 256, 512])
def test_cuda_core_kernel_at_other_dimensions(dim, monkeypatch):
    """k_nn2 (dim 128 only with TBM_PATH=exact; from 176 on, dynamic + static shared memory pass the 48 KB a launch gets by default)"""
    monkeypatch.setenv("TBM_PATH", "exact")
    rng = np.random.default_rng(dim)
    n = (45, 70, 33) if not _emulated() else (20, 37, 9)
    base = rng.normal(size=(max(n), dim)).astype(np.float32)
    sets = [np.ascontiguousarray(base[rng.permutation(max(n))[:k]] + 0.1 * rng.normal(size=(k, dim)).astype(np.float32)) for k in n]
    sets[1][5] = sets[1][9]   # duplicate rows: exact ties
    pairs = [(0, 1), (1, 0), (1, 2), (2, 2)]
    _check_nn2(sets, pairs, ("dim", dim))
    _check_match_all(sets, pairs, ("dim", dim), option_sets=OPTION_SETS[:2])


def test_dimension_limits():
    for dim in (0, 513):
        sets = [np.zeros((3, dim), np.float32), np.zeros((4, dim), np.float32)]
        rc, _, _ = matcher.match_all(sets, [(0, 1)])
        assert rc == -1, (dim, rc)


# ------------------------------------------------------------------ host loops at scale (tensor-core path against the CUDA-core path)
scale = pytest.mark.skipif(_emulated(), reason="millions of queries: hours under the SIMT emulator")


def _sift_like(rng, n, n_shared=None, base=None):
    s = np.abs(rng.normal(size=(n, 128))).astype(np.float32)
    if base is not None:
        s[:n_shared] = base[rng.permutation(len(base))[:n_shared]] + 0.05 * np.abs(rng.normal(size=(n_shared, 128))).astype(np.float32)
    return np.ascontiguousarray(s / np.linalg.norm(s, axis=1, keepdims=True), np.float32)


@scale
def test_two_chunks_of_queries(monkeypatch):
    """1100 repeats of one pair of 2048-descriptor images = 4.5 M queries: the tensor-core path splits them into two chunks (4 M
    queries each at most); every repeat gives the same list, the CUDA-core path's list, and the oracle's on both sides of the boundary"""
    rng = np.random.default_rng(24)
    base = np.abs(rng.normal(size=(1800, 128))).astype(np.float32)
    sets = [_sift_like(rng, 2048, 1600, base), _sift_like(rng, 2048, 1600, base)]
    pairs = [(0, 1)] * 1100
    per_chunk = (4 << 20) // 4096
    assert per_chunk < len(pairs)
    opt = matcher.default_options()
    out = {}
    for path in ("tc", "exact"):
        _set_path(monkeypatch, path)
        rc, moff, ok, arr = _raw_match_all(sets, pairs, opt, 1100 * 2048)
        assert rc == 0
        out[path] = (moff, ok, arr[:int(moff[-1])])
    moff, ok, arr = out["tc"]
    assert np.array_equal(moff, out["exact"][0]) and np.array_equal(ok, out["exact"][1]) and np.array_equal(arr, out["exact"][2])
    counts = np.diff(moff)
    assert np.all(counts == counts[0]) and counts[0] > 1000 and ok.all()
    first = arr[:counts[0]]
    for p in range(len(pairs)):
        assert np.array_equal(arr[moff[p]:moff[p + 1]], first), p
    ok_o, exp = _oracle_match(sets[0], sets[1])
    for p in (per_chunk - 1, per_chunk):
        got = [(int(m["i"]), int(m["j"]), float(m["d"])) for m in arr[moff[p]:moff[p + 1]]]
        assert bool(ok[p]) == ok_o and got == exp, p


@scale
def test_many_pairs_and_segments(monkeypatch):
    """5000 pairs of small images (> 4096: k_pair_decide / k_gather_matches loop over their capped grid) = 10000 query segments
    (> 8192: k_expand_segments loops), pairs with an empty image among them"""
    rng = np.random.default_rng(25)
    sets = [_sift_like(rng, int(n)) for n in rng.integers(1, 9, 120)] + [np.zeros((0, 128), np.float32)]
    sets[7] = np.ascontiguousarray(sets[3][::-1])
    pairs = [(int(a), int(b)) for a, b in rng.integers(0, len(sets), size=(5000, 2))]
    opt = matcher.default_options(min_num_feature_matches=1)
    out = {}
    for path in ("tc", "exact"):
        _set_path(monkeypatch, path)
        rc, moff, ok, arr = _raw_match_all(sets, pairs, opt, 50000)
        assert rc == 0
        out[path] = (moff, ok, arr[:int(moff[-1])])
    for a, b in zip(out["tc"], out["exact"]):
        assert np.array_equal(a, b)
    moff, ok, arr = out["exact"]
    assert ok.sum() > 10 and (~ok.astype(bool)).sum() > 10
    for p in range(0, len(pairs), 97):
        ok_o, exp = _oracle_match(sets[pairs[p][0]], sets[pairs[p][1]], min_num_feature_matches=1)
        got = [(int(m["i"]), int(m["j"]), float(m["d"])) for m in arr[moff[p]:moff[p + 1]]]
        assert bool(ok[p]) == ok_o and got == exp, p
