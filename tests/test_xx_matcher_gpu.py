"""Secondary path on the GPU: tbm_match_all (CUDA-core round-1 kernel, bit-exact float summation order) against the CPU
oracle -- identical match lists including distances -- on the reference's three matcher cases and on random unit
descriptors (SIFT-like 128-D, ragged image sizes).  First executed by the round-end driver (GPU budget, DESIGN.md 7.4)."""
import numpy as np
import pytest

from test_matcher_host import _oracle_match
from theiasfm_b200 import matcher

pytestmark = pytest.mark.gpu


def _unit(v):
    v = np.asarray(v, np.float32)
    return v / np.linalg.norm(v)


def test_reference_cases_on_gpu():
    ones = np.stack([_unit(np.ones(10))] * 10)
    a = np.ones(10, np.float32); a[0] = 0.9
    b = np.ones(10, np.float32); b[0] = 0.89
    c = np.ones(10, np.float32); c[0] = 0
    d = np.ones(10, np.float32); d[1] = 0; d[2] = 0
    sets = [ones, ones.copy(), _unit(np.ones(10))[None], np.stack([_unit(a), _unit(b)]),
            np.stack([_unit(np.ones(10)), np.eye(10, dtype=np.float32)[0]]), np.stack([_unit(c), _unit(d)])]
    for pair, kw in (((0, 1), dict(min_num_feature_matches=0, keep_only_symmetric_matches=0, use_lowes_ratio=0)),
                     ((2, 3), dict(min_num_feature_matches=0, keep_only_symmetric_matches=0, use_lowes_ratio=1)),
                     ((4, 5), dict(min_num_feature_matches=0, keep_only_symmetric_matches=1, use_lowes_ratio=0))):
        rc, res, ok = matcher.match_all(sets, [pair], matcher.default_options(**kw))
        ok_o, exp = _oracle_match(np.ascontiguousarray(sets[pair[0]]), np.ascontiguousarray(sets[pair[1]]), **kw)
        assert rc == 0 and ok[0] == ok_o and res[0] == exp
    assert len(res[0]) == 1  # the reference's SymmetricMatches expectation


def test_random_descriptors_match_oracle_exactly():
    rng = np.random.default_rng(77)
    base = rng.normal(size=(700, 128)).astype(np.float32)
    sets = []
    for n in (700, 513, 31, 1000, 2):
        take = base[rng.permutation(700)[:min(n, 700)]] + 0.05 * rng.normal(size=(min(n, 700), 128)).astype(np.float32)
        extra = rng.normal(size=(max(0, n - 700), 128)).astype(np.float32)
        s = np.concatenate([take, extra]).astype(np.float32)
        sets.append(np.ascontiguousarray(s / np.linalg.norm(s, axis=1, keepdims=True)))
    pairs = [(0, 1), (1, 0), (0, 3), (2, 3), (3, 4), (4, 2), (1, 1)]
    for kw in (dict(), dict(keep_only_symmetric_matches=0), dict(use_lowes_ratio=0, min_num_feature_matches=0)):
        rc, res, ok = matcher.match_all(sets, pairs, matcher.default_options(**kw))
        assert rc == 0
        for p, (i, j) in enumerate(pairs):
            ok_o, exp = _oracle_match(sets[i], sets[j], **kw)
            assert ok[p] == ok_o and res[p] == exp, (kw, i, j)
    assert sum(len(r) for r in res) > 1000


def test_tensor_core_path_equals_the_exact_kernel_at_sift_size(monkeypatch):
    """dim 128 goes through the wgmma / TMA candidate pass + exact re-evaluation (tbm_matcher_tc.cuh); TBM_PATH=exact forces the
    round-1 CUDA-core kernel (bit-exact float order), the checker here: the match lists -- indices AND distances -- must be identical
    at SIFT-like sizes (non-negative unit descriptors, thousands per image, sizes that are not multiples of the 128-row tiles), with
    and without the ratio test, including an image matched against itself (zero distances, exact ties)."""
    rng = np.random.default_rng(5)
    base = np.abs(rng.normal(size=(3000, 128))).astype(np.float32)
    sets = []
    for n in (3000, 2500, 129, 4097):
        idx = rng.permutation(3000)[:min(n, 3000)]
        s = base[idx] + 0.08 * np.abs(rng.normal(size=(len(idx), 128))).astype(np.float32)
        if n > 3000:
            s = np.concatenate([s, np.abs(rng.normal(size=(n - 3000, 128))).astype(np.float32)])
        sets.append(np.ascontiguousarray(s / np.linalg.norm(s, axis=1, keepdims=True), np.float32))
    sets[2][7] = sets[2][3]  # duplicate descriptors: equal distances, the lower index must win
    pairs = [(0, 1), (1, 0), (0, 3), (2, 3), (3, 2), (2, 2), (1, 1)]
    for kw in (dict(), dict(use_lowes_ratio=0, min_num_feature_matches=0, keep_only_symmetric_matches=0)):
        monkeypatch.delenv("TBM_PATH", raising=False)
        rc_t, res_t, ok_t = matcher.match_all(sets, pairs, matcher.default_options(**kw))
        monkeypatch.setenv("TBM_PATH", "exact")
        rc_e, res_e, ok_e = matcher.match_all(sets, pairs, matcher.default_options(**kw))
        assert rc_t == 0 and rc_e == 0 and ok_t == ok_e
        for p in range(len(pairs)):
            assert res_t[p] == res_e[p], (kw, pairs[p], len(res_t[p]), len(res_e[p]))
    assert sum(len(r) for r in res_t) > 5000


def test_exact_pass_with_overflowed_queries_equals_the_sequential_scan():
    """k_exact_top2 alone (tbm_debug_exact_top2) on hand-made candidate lists: queries whose lists hold the true two nearest plus decoys,
    queries flagged as overflowed in either column half (scanned exhaustively by the whole CTA through shared memory: candidate counts
    that are not multiples of the 64-row tiles, several overflowed queries in one CTA, an image with a single descriptor), duplicate rows
    (equal distances: the lower index wins).  Reference: float32 accumulation term by term without FMA (distance.h:52-56)."""
    from test_matcher_host import _nn2_float32
    rng = np.random.default_rng(11)
    nA, nB, nC = 70, 333, 1
    D = np.abs(rng.normal(size=(nA + nB + nC, 128))).astype(np.float32)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    D[nA + 200] = D[nA + 17]                                 # duplicate candidate rows
    A, B, Cc = D[:nA], D[nA:nA + nB], D[nA + nB:]
    bj, bd, sd = _nn2_float32(A, B)
    order = np.argsort(((A[:, None, :] - B[None, :, :]) ** 2).sum(-1), axis=1, kind="stable")
    q_row = np.arange(nA, dtype=np.int32)
    b_row0 = np.full(nA, nA, np.int32); b_rows = np.full(nA, nB, np.int32)
    cand = np.full((nA, 16), -1, np.int32)
    for i in range(nA):
        true2 = order[i, :2] + nA
        decoys = rng.choice(nB, 5, replace=False) + nA
        slots = rng.permutation(16)[:7]
        cand[i, slots] = np.concatenate([true2, decoys])
    cand[10, :] = -1                                         # a query without candidates (the other image was empty in pass 1)
    bj[10], bd[10], sd[10] = -1, 0.0, 0.0
    cand[11, :] = -1; cand[11, 15] = order[11, 0] + nA       # a single candidate, in the last slot: no runner-up
    bj[11], bd[11], sd[11] = order[11, 0], bd[11], 0.0
    ovf = [3, 5, 6, 31, 32, 40, 69]                          # 3, 5, 6, 31: four overflowed queries in the first CTA
    for k, i in enumerate(ovf):
        cand[i, :] = -1
        cand[i, 0 if k % 2 == 0 else 8] = -2
    # the last query runs against the one-descriptor image
    q_row = np.concatenate([q_row, [5]]).astype(np.int32); b_row0 = np.concatenate([b_row0, [nA + nB]]).astype(np.int32)
    b_rows = np.concatenate([b_rows, [1]]).astype(np.int32)
    last = np.full((1, 16), -1, np.int32); last[0, 8] = -2
    cand = np.concatenate([cand, last])
    rc, gj, gd, gs = matcher.exact_top2(D, q_row, b_row0, b_rows, cand)
    assert rc == 0
    assert np.array_equal(gj[:nA], bj) and np.array_equal(gd[:nA], bd) and np.array_equal(gs[:nA], sd)
    j1, d1, _ = _nn2_float32(A[5:6], Cc)
    assert gj[nA] == 0 and gd[nA] == d1[0] and gs[nA] == 0.0
