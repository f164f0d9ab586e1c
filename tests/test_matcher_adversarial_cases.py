"""CPU side of the adversarial matcher cases (tests/matcher_cases.py): the cases really are adversarial, and the numpy model of
k_nn_candidates' selection rule keeps the reference's two nearest neighbours in every one of them -- while a rule with a quarter of
the margin, or the rule before the score interval (strict comparison against the runner-up's score, no norm term), misses some.
The model guides the kernel's margin; the GPU tests (test_xx_matcher_gpu_adversarial.py) check the kernel itself."""
import numpy as np
import pytest

import matcher_cases as mc


def test_tie_groups_are_adversarial():
    """classes C and D: for the query x the reference's three nearest distances (float64) lie closer together than the TF32 error of
    their scores (2^-9 sum_k |x_k y_k| each way for round-to-nearest operands, 2^-8 for truncated ones): TF32 alone cannot rank them"""
    for cls, (name, sets, _) in mc.all_cases():
        if cls not in "CD":
            continue
        Q, C = sets[0].astype(np.float64), sets[1].astype(np.float64)
        x = Q[0]
        d = ((C - x) ** 2).sum(1)
        s, order = mc.reference_order(sets[0][:1], sets[1])
        top3 = order[0, :3]
        tf32_err = 2.0 ** -9 * np.abs(C[top3] * x).sum(1).max()
        assert np.ptp(d[top3]) < tf32_err, (name, d[top3], tf32_err)


@pytest.mark.parametrize("cls", sorted(mc.CLASSES))
def test_shipped_rule_keeps_the_reference_top2(cls):
    for name, sets, pairs in mc.CLASSES[cls]():
        nonneg = mc.call_is_nonneg(sets)
        for Q, C in mc.directions(sets, pairs):
            if len(Q) and len(C):
                miss = mc.model_misses(Q, C, nonneg, mc.shipped_rule(nonneg))
                assert len(miss) == 0, (name, miss)


@pytest.mark.parametrize("cls", sorted(mc.CLASSES))
def test_weaker_rules_miss(cls):
    """the test's own teeth: with a quarter of the margin the model drops a reference top-2 element in some case of every class
    with a TF32 term (class B has x.y = 0: nothing for the TF32 margin to cover), and the rule before the interval (strict '<',
    no norm term) does so in every class"""
    quarter = parent = 0
    for name, sets, pairs in mc.CLASSES[cls]():
        nonneg = mc.call_is_nonneg(sets)
        for Q, C in mc.directions(sets, pairs):
            if len(Q) and len(C):
                quarter += len(mc.model_misses(Q, C, nonneg, mc.shipped_rule(nonneg, 0.25)))
                parent += len(mc.model_misses(Q, C, nonneg, mc.parent_rule()))
    assert parent > 0
    if cls != "B":
        assert quarter > 0


def test_classes_cover_both_margins_and_exact_ties():
    cases = mc.all_cases()
    assert {cls for cls, _ in cases} == set("ABCDE")
    kinds = {(cls, mc.call_is_nonneg(sets)) for cls, (_, sets, _) in cases}
    assert ("A", True) in kinds and ("A", False) in kinds and ("D", False) in kinds
    # the reference's own ties: the zero candidates (distance 0 from a zero query, ||x||^2 from x, like 2x) and duplicated byte rows
    for cls, (name, sets, _) in cases:
        if cls == "A":
            s, order = mc.reference_order(sets[0][:2], sets[1])
            assert s[0, order[0, 0]] == s[0, order[0, 1]] == 0.0
            assert s[1, 0] == s[1, 1] == s[1, 2]   # 2x and the two zero rows: bit-identical reference distances


def test_truncation_probe_tells_truncation_from_rounding():
    """the GPU test test_tf32_operands_are_truncated reads the hardware's TF32 conversion off this probe: under truncation the
    query keeps two candidates, under round-to-nearest all 18 (exhaustive scan)"""
    Q, C = mc.truncation_probe()
    rule = mc.shipped_rule(True)
    assert mc.model_lists(Q, C, True, rule).sum() == 2
    assert mc.model_lists(Q, C, True, rule, rounding=True).sum() == 18
    assert len(mc.model_misses(Q, C, True, rule)) == 0


def test_model_constants_are_the_kernels():
    """the model uses k_nn_candidates' own float constants (read from the source), and each is the float32 value of the margin
    formula rounded away from the tighter side"""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "theiasfm_b200", "csrc", "tbm_matcher_tc.cuh")).read()
    for key in ("kLo", "kUp", "kK", "kX"):
        m = re.search(r"constexpr float %s = NONNEG \? (\S+)f : (\S+)f;" % key, src)
        assert m, key
        assert float.fromhex(m.group(1)) == mc.KERNEL_CONSTANTS[True][key]
        assert float.fromhex(m.group(2)) == mc.KERNEL_CONSTANTS[False][key]
    for nonneg, k in mc.KERNEL_CONSTANTS.items():
        ideal = mc.shipped_rule(nonneg, scale=1.0 - 1e-15)   # the formula in float64
        for key, v in k.items():
            assert float(np.float32(v)) == v
            assert (abs(v) <= abs(ideal[key])) if key == "kUp" else (abs(v) >= abs(ideal[key])), (nonneg, key)
            assert abs(v - ideal[key]) <= 2.0 ** -22 * abs(v)
