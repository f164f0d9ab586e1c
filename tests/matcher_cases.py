"""Seeded adversarial inputs for the matcher's TF32 candidate pass (k_nn_candidates) and a numpy model of its selection rule.

Every generator returns a list of cases (name, descriptor sets, pairs); all descriptors are 128-dimensional float32, so the
tensor-core path takes them.  The classes:
  A  zero query rows and zero candidate rows (exact ties at distance 0 and at distance ||x||^2), in a call whose descriptors are
     all >= 0 and in a call where another image has one negative component (which selects the general margin for the whole call);
  B  sparse non-negative descriptors with disjoint supports (x.y = 0 exactly), candidates permutations of one multiset of values:
     the true distances are equal and only the reference's float rounding orders them;
  C  near-ties below TF32 resolution: a query whose components lose the most to TF32 (all 13 dropped mantissa bits set, or the
     pattern that rounds up the most), candidates 2x, x + u (u on the complementary support) and a short candidate at the same
     distance, with unit norms and with norm ratios up to 10^3 between the near-tied candidates;
  D  signed descriptors, same construction: the runner-up 2x has ||y||^2 = 4 ||x||^2, much more than ||x||^2 + ||y_n||^2 of the
     zero candidate it ties with;
  E  integer-valued descriptors 0..255 (raw-byte SIFT: every product and sum is exact in float, masses of exact ties, the lower index
     must win) and the class-C construction scaled by 2^-10 and 2^10.
"""
import numpy as np

DIM = 128
TRUNC, ROUND_UP = 0x1FFF, 0x1001   # low-13-bit patterns: the largest truncation loss / the largest round-to-nearest gain


def coherent(rng, n_comp, pattern, exps=(3, 4), signed=False):
    """n_comp float32 values 2^-e (1 + 2^-23 pattern): top mantissa bits zero, so the TF32 operand error is the largest
    relative error the pattern allows (2^-10 for TRUNC under truncation, 2^-11 for ROUND_UP under rounding)."""
    e = rng.choice(exps, n_comp)
    bits = ((127 - e).astype(np.uint32) << 23) | np.uint32(pattern)
    if signed:
        bits |= (rng.random(n_comp) < 0.5).astype(np.uint32) << 31
    return bits.view(np.float32)


def far_rows(rng, n, x_norm2, signed=False):
    """filler rows at distance >= 9 ||x||^2 from every query of norm^2 <= ||x||^2 (norm 4 ||x||): they never tie the near group"""
    v = rng.normal(size=(n, DIM))
    if not signed:
        v = np.abs(v)
    v *= 4.0 * np.sqrt(max(x_norm2, 1e-30)) / np.linalg.norm(v, axis=1, keepdims=True)
    return v.astype(np.float32)


def _norm2(v):
    return float(np.dot(v.astype(np.float64), v.astype(np.float64)))


def _tie_group(rng, pattern, signed, norm_ratio=None, scale=1.0):
    """query x (support = first 64 dimensions) and candidates at distance ~ ||x||^2 from it:
    2x (exactly the reference distance of the zero vector: x - 2x = -x), two zero rows, x + u with u on the other 64 dimensions and
    ||u||^2 within 2^-14 of ||x||^2, and, with norm_ratio, a short candidate mu x + v of norm^2 4 ||x||^2 / norm_ratio at the same distance."""
    x = np.zeros(DIM, np.float32)
    x[:64] = coherent(rng, 64, pattern, signed=signed)
    x *= np.float32(scale)
    X = _norm2(x)
    cands = [2 * x, np.zeros(DIM, np.float32), np.zeros(DIM, np.float32)]
    for _ in range(2):
        u = np.zeros(DIM)
        u[64:] = rng.normal(size=64) if signed else np.abs(rng.normal(size=64))
        u *= np.sqrt(X) / np.linalg.norm(u)
        cands.append((x.astype(np.float64) + u).astype(np.float32))
    if norm_ratio:
        mu = 2.0 / norm_ratio
        v = np.zeros(DIM)
        v[64:] = rng.normal(size=64) if signed else np.abs(rng.normal(size=64))
        v *= np.sqrt(X * (2 * mu - mu * mu)) / np.linalg.norm(v)
        cands.append((mu * x.astype(np.float64) + v).astype(np.float32))
    return x, np.stack(cands), X


def _with_fillers(rng, rows, n_fill, X, signed):
    return np.ascontiguousarray(np.concatenate([rows, far_rows(rng, n_fill, X, signed)]).astype(np.float32))


def class_a(seed=1):
    rng = np.random.default_rng(seed)
    cases = []
    for signed_call in (False, True):
        x, cands, X = _tie_group(rng, TRUNC, signed=False)
        Q = _with_fillers(rng, np.stack([np.zeros(DIM, np.float32), x, 0.5 * x]), 5, X, False)
        C = _with_fillers(rng, cands, 70, X, False)                       # 75 rows: two tiles
        Z = np.zeros((3, DIM), np.float32)                                # an image of zero rows only
        sets = [Q, C, Z]
        if signed_call:
            neg = far_rows(rng, 4, X)
            neg[2, 17] = -neg[2, 17]                                      # one negative component in the whole call
            sets.append(np.ascontiguousarray(neg))
        cases.append(("A-%s" % ("signed-call" if signed_call else "nonneg"), sets, [(0, 1), (1, 0), (0, 2), (2, 1), (2, 2)]))
    return cases


def class_b(seed=2):
    rng = np.random.default_rng(seed)
    cases = []
    for k, n_support in enumerate((8, 24, 64)):
        qv = np.abs(rng.normal(size=n_support)).astype(np.float32)
        cv = np.abs(rng.normal(size=n_support)).astype(np.float32) * np.float32(1.0 + 0.37 * k)
        Q = np.zeros((6, DIM), np.float32)
        for i in range(len(Q)):
            Q[i, rng.permutation(64)[:n_support]] = rng.permutation(qv)      # supports inside [0, 64)
        C = np.zeros((70, DIM), np.float32)
        for i in range(len(C)):
            C[i, 64 + rng.permutation(64)[:n_support]] = rng.permutation(cv)  # supports inside [64, 128): disjoint from every query
        cases.append(("B-support%d" % n_support, [Q, C], [(0, 1), (1, 0)]))
    return cases


def class_c(seed=3):
    rng = np.random.default_rng(seed)
    cases = []
    for pattern, pname in ((TRUNC, "trunc"), (ROUND_UP, "round")):
        for ratio in (None, 10.0, 1e3):
            x, cands, X = _tie_group(rng, pattern, signed=False, norm_ratio=ratio)
            Q = _with_fillers(rng, np.stack([x]), 3, X, False)
            C = _with_fillers(rng, cands, 60, X, False)
            cases.append(("C-%s-ratio%s" % (pname, "1" if ratio is None else "%g" % ratio), [Q, C], [(0, 1), (1, 0)]))
    return cases


def class_d(seed=4):
    rng = np.random.default_rng(seed)
    cases = []
    for pattern, pname in ((TRUNC, "trunc"), (ROUND_UP, "round")):
        for ratio in (None, 1e3):
            x, cands, X = _tie_group(rng, pattern, signed=True, norm_ratio=ratio)
            Q = _with_fillers(rng, np.stack([x, -x, np.zeros(DIM, np.float32)]), 3, X, True)
            C = _with_fillers(rng, cands, 66, X, True)
            cases.append(("D-%s-ratio%s" % (pname, "1" if ratio is None else "%g" % ratio), [Q, C], [(0, 1), (1, 0)]))
    return cases


def class_e(seed=5):
    rng = np.random.default_rng(seed)
    # raw-byte SIFT: few distinct values, duplicated rows, a zero row; everything exact in float and in TF32
    base = rng.integers(0, 4, size=(40, DIM)).astype(np.float32) * np.float32(85)
    Q = base[rng.integers(0, 40, 50)].copy(); Q[3] = 0
    C = np.concatenate([base[rng.integers(0, 40, 90)], rng.integers(0, 256, size=(40, DIM)).astype(np.float32)])
    C[5] = 0; C[77] = C[12]
    cases = [("E-bytes", [np.ascontiguousarray(Q), np.ascontiguousarray(C)], [(0, 1), (1, 0), (1, 1)])]
    for scale, sname in ((2.0 ** -10, "2^-10"), (2.0 ** 10, "2^10")):
        x, cands, X = _tie_group(rng, TRUNC, signed=False, norm_ratio=10.0, scale=scale)
        Qs = _with_fillers(rng, np.stack([x, np.zeros(DIM, np.float32)]), 3, X, False)
        Cs = _with_fillers(rng, cands, 60, X, False)
        cases.append(("E-scaled-%s" % sname, [Qs, Cs], [(0, 1), (1, 0)]))
    return cases


CLASSES = {"A": class_a, "B": class_b, "C": class_c, "D": class_d, "E": class_e}


def all_cases():
    return [(cls, c) for cls, gen in CLASSES.items() for c in gen()]


# ------------------------------------------------------------------ numpy model of the selection rule of k_nn_candidates
def tf32(a, rounding=False):
    """wgmma .tf32 operand: the low 13 mantissa bits dropped (truncation), or rounded to nearest (what the margin does NOT assume)"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    if rounding:
        u = u + np.uint32(0x1000)
    return (u & np.uint32(0xFFFFE000)).view(np.float32)


def truncation_probe(seed=6):
    """query x (TRUNC pattern: each operand loses ~2^-10 to truncation, ~2^-23 to rounding), candidates: two zero rows at distance
    ||x||^2, then 16 rows 2x + v_i e_(64+i) at distance ||x||^2 + 2^-8 ||x||^2.  Truncation over-estimates the scores of the 2x rows
    by ~2^-7 ||x||^2, which puts them outside the interval of the zero rows: the query keeps a 2-entry list.  Rounding would keep all
    18 rows (more than the 16 slots): the query would be scanned exhaustively."""
    rng = np.random.default_rng(seed)
    x = np.zeros(DIM, np.float32)
    x[:64] = coherent(rng, 64, TRUNC)
    X = _norm2(x)
    rows = [np.zeros(DIM, np.float32), np.zeros(DIM, np.float32)]
    for i in range(16):
        y = 2 * x
        y[64 + i] = np.float32(np.sqrt(2.0 ** -8 * X))
        rows.append(y)
    return np.ascontiguousarray(x[None]), np.ascontiguousarray(np.stack(rows))


def row_norms(d):
    """k_row_norms: float, four squares at a time, left to right"""
    d = np.asarray(d, np.float32)
    s = np.zeros(len(d), np.float32)
    for k in range(0, DIM, 4):
        t = d[:, k] * d[:, k] + d[:, k + 1] * d[:, k + 1] + d[:, k + 2] * d[:, k + 2] + d[:, k + 3] * d[:, k + 3]
        s = (s + t).astype(np.float32)
    return s


def _f32(v):
    return np.asarray(v, np.float64).astype(np.float32)


# the shipped rule (k_nn_candidates): lo' = fmaf(kLo, acc, Y), up' = fmaf(kUp, acc, Y), keep lo' <= fmaf(u2', kK, kX X)
# with u2' the second smallest up' of the row -- the interval [lo, up] of the kernel's comment, scaled by 1 / (1 -+ b)
MARGINS = {True: dict(b=2.0 ** -16, a_lo=2.0 ** -8 + 2.0 ** -14, a_up=2.0 ** -14),
           False: dict(b=2.0 ** -9 + 2.0 ** -13, a_lo=0.0, a_up=0.0)}
_H = float.fromhex
KERNEL_CONSTANTS = {True: dict(kLo=_H("-0x1.008302p+1"), kUp=_H("-0x1.fffap+0"), kK=_H("0x1.000202p+0"), kX=_H("0x1.000102p-15")),
                    False: dict(kLo=_H("-0x1.00884ap+1"), kUp=_H("-0x1.fef09p+0"), kK=_H("0x1.011092p+0"), kX=_H("0x1.1090cep-8"))}


def shipped_rule(nonneg, scale=1.0):
    """the kernel's constants; scale != 1 multiplies every margin term (b and both TF32 coefficients) -- a weaker rule for scale < 1"""
    if scale == 1.0:
        return dict(kind="interval", **KERNEL_CONSTANTS[nonneg])
    m = {k: v * scale for k, v in MARGINS[nonneg].items()}
    b = m["b"]
    return dict(kind="interval", kLo=-(2 + m["a_lo"]) / (1 - b), kUp=-(2 - m["a_up"]) / (1 + b), kK=(1 + b) / (1 - b), kX=2 * b / (1 - b))


def parent_rule():
    """the rule before the interval: val = score - margin_n < runner-up score (+ 2^-8 ||x||^2 with signed descriptors)"""
    return dict(kind="parent")


def model_lists(Q, C, nonneg, rule, rounding=False):
    """boolean [len(Q), len(C)]: the candidates the rule hands to the exact pass (before the 16-slot limit)"""
    acc = _f32(tf32(Q, rounding).astype(np.float64) @ tf32(C, rounding).astype(np.float64).T)
    nn = row_norms(C)[None, :].astype(np.float64)
    X = row_norms(Q)[:, None].astype(np.float64)
    a = acc.astype(np.float64)
    if rule["kind"] == "parent":
        sc = _f32(nn - 2.0 * a).astype(np.float64)
        if nonneg:
            val = _f32(sc - (2.0 ** -8 + 2.0 ** -14) * a)
            lim_add = 0.0
        else:
            val = _f32(sc - 2.0 ** -8 * nn)
            lim_add = _f32(2.0 ** -8 * X)
        r2 = np.sort(sc, axis=1)[:, 1:2] if C.shape[0] > 1 else np.full((len(Q), 1), np.inf)
        return val < _f32(r2 + lim_add)
    f = lambda v: np.float64(np.float32(v))
    lo = _f32(nn + f(rule["kLo"]) * a)
    up = _f32(nn + f(rule["kUp"]) * a)
    u2 = np.sort(up, axis=1)[:, 1:2].astype(np.float64) if C.shape[0] > 1 else np.full((len(Q), 1), 2.0 ** 126)
    lim = _f32(u2 * f(rule["kK"]) + f(rule["kX"]) * X)
    return lo <= lim


def reference_order(Q, C):
    """the reference's float distances (left to right, no FMA) and the candidate order (distance, then index)"""
    s = np.zeros((len(Q), len(C)), np.float32)
    for k in range(DIM):
        d = (Q[:, None, k] - C[None, :, k]).astype(np.float32)
        s = (s + (d * d).astype(np.float32)).astype(np.float32)
    return s, np.argsort(s, axis=1, kind="stable")


def model_misses(Q, C, nonneg, rule, kc=16):
    """queries whose reference top-2 is not in the rule's list (a list longer than kc is scanned exhaustively: never a miss)"""
    keep = model_lists(Q, C, nonneg, rule)
    _, order = reference_order(Q, C)
    top = order[:, :min(2, C.shape[0])]
    ok = np.take_along_axis(keep, top, axis=1).all(axis=1) | (keep.sum(axis=1) > kc)
    return np.flatnonzero(~ok)


def directions(sets, pairs):
    """(query set, candidate set) of every direction the symmetric matcher evaluates"""
    for a, b in pairs:
        yield sets[a], sets[b]
        yield sets[b], sets[a]


def call_is_nonneg(sets):
    return all(float(np.min(s)) >= 0.0 for s in sets if len(s))
