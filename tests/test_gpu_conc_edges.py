"""GPU: the concordance counters and precision-recall curves of csrc/concordance.cu at their edges.

Every float is compared as its uint64 bit pattern.  The reference is the reference's own output (golden) for the
frames of make_edge_cases / make_error_cases, and an exact restatement written here for ConcordanceContext.run +
curve: int64 counts at each distinct score, correctly rounded fp64 quotients, and the threshold of a run of equal
scores taken from its first element in input order (scikit-learn 1.5, the reference's pin)."""
from fractions import Fraction

import numpy as np
import pytest

from tests.concordance_data import extreme_family, ulp_family
from tests.test_concordance_cpu import (EDGE_CASES, SIGNED_ZERO_KATS, assert_bits_equal, check_against_golden,
                                        load_golden)
from variantcalling_b200 import concordance as PC
from variantcalling_b200 import lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = PC.ConcordanceContext(0)
    yield c
    c.close()


def exact_curve(scores, truth):
    """The raw curve of one selection: (precision, recall, thresholds) in increasing-threshold order, and the int64
    true / false positive counts at each distinct score in decreasing order."""
    order = np.argsort(-scores, kind="stable")  # decreasing; equal scores (-0.0 with +0.0) keep their input order
    s, t = scores[order], truth[order].astype(np.int64)
    ends = np.r_[np.flatnonzero(s[1:] != s[:-1]), len(s) - 1]
    starts = np.r_[0, ends[:-1] + 1]
    tps = np.cumsum(t)[ends]
    fps = ends + 1 - tps
    precision = tps / (tps + fps)  # int64 -> fp64 is exact below 2^53: one correctly rounded division
    recall = np.ones(len(tps)) if tps[-1] == 0 else tps / tps[-1]
    return precision[::-1], recall[::-1], s[starts][::-1], tps, fps


def check_fraction_sample(tps, fps, p, r, rng, k=64):
    """A sample of the quotients against exact rationals (Fraction -> float rounds correctly)."""
    d = len(tps)
    for i in rng.choice(d, size=min(k, d), replace=False):
        o = d - 1 - i
        assert_bits_equal(p[o], float(Fraction(int(tps[i]), int(tps[i] + fps[i]))), f"precision at {i}")
        if tps[-1]:
            assert_bits_equal(r[o], float(Fraction(int(tps[i]), int(tps[-1]))), f"recall at {i}")


def labels(rng, n, p_fn=0.05):
    """cls codes (0 fp, 1 tp, 2 fn, 3 tn) and calls."""
    cls = np.where(rng.random(n) < 0.6, 1, 0).astype(np.uint8)
    cls[rng.random(n) < 0.03] = 3
    cls[rng.random(n) < p_fn] = 2
    return cls, (rng.random(n) < 0.7).astype(np.uint8)


def expected_counts(scores, pred, cls, member):
    """The 8 counters of one group: the six metric counters, then NaN and inf scores of called records."""
    called = member & (cls != 2)
    truth = (cls == 1) | (cls == 2)
    t, p, s = truth[called], pred[called] != 0, scores[called]
    return np.array([(t & p).sum(), (p & ~t).sum(), (~p & t).sum(), t.sum(), called.sum(), (member & (cls == 2)).sum(),
                     np.isnan(s).sum(), np.isinf(s).sum()], np.int64)


def check_counts(res, want, what):
    """want: (9, 8), the device's counter block; ConcordanceContext.run splits it into counts and non_finite."""
    np.testing.assert_array_equal(res["counts"], want[:, :6], err_msg=what)
    np.testing.assert_array_equal(res["non_finite"], want[:, 6:], err_msg=what)


def check_one_group(ctx, scores, cls, pred, rng, what):
    """Everything in group 0 (given ids): counts, selection, cutoff and the raw curve against the exact reference."""
    n = len(scores)
    res = ctx.run(scores, pred, cls, np.zeros(n, np.uint8), np.zeros(n, np.int32), group=np.zeros(n, np.int8))
    want = np.zeros((9, 8), np.int64)
    want[0] = expected_counts(scores, pred, cls, np.ones(n, bool))
    check_counts(res, want, what)
    called = cls != 2
    s, t = scores[called], (cls[called] == 1)
    np.testing.assert_array_equal(res["selected"][0], [called.sum(), t.sum()], err_msg=what)
    if not called.any():
        assert res["curve_len"][0] == 0
        return
    p, r, thr, tps, fps = exact_curve(s, t)
    assert res["curve_len"][0] == len(thr), what
    # the 20th largest score in the stable decreasing order (only compared against, so a zero's sign is moot for the
    # curve; the stable order pins it all the same)
    assert_bits_equal(res["cutoff"][0], s[np.argsort(-s, kind="stable")][min(len(s) - 1, 19)], f"{what}: cutoff")
    gp, gr, gt = ctx.curve(0, len(thr))
    assert_bits_equal(gp, p, f"{what}: precision")
    assert_bits_equal(gr, r, f"{what}: recall")
    assert_bits_equal(gt, thr, f"{what}: thresholds")
    check_fraction_sample(tps, fps, gp, gr, rng)


def score_families(rng):
    n = 3000
    yield "mixed_sign_ties", np.round(rng.normal(0, 4, n), 1)  # signed zeros included
    yield "distinct_negative", -rng.permutation(n).astype(np.float64) - 0.5
    yield "ulp_apart", rng.choice(ulp_family(), n)
    yield "subnormal_and_huge", rng.choice(extreme_family(), n)
    yield "single_score", np.full(n, -7.25)
    z = np.where(rng.random(n) < 0.5, -0.0, 0.0)
    for first, tag in ((-0.0, "neg"), (0.0, "pos")):  # a run of signed zeros that starts with either sign
        yield f"zeros_first_{tag}", np.concatenate([[first], z, [1.0, -1.0]])
    yield "cutoff_in_a_tie", np.array([4.0] * 18 + [2.0, 2.0, 1.0])  # the 20th largest score sits in a tie run


@pytest.mark.parametrize("order", ["shuffled", "ascending", "descending"])
def test_run_and_curve_match_the_exact_reference_over_score_families(ctx, order):
    rng = np.random.default_rng(5)
    for name, s in score_families(rng):
        s = np.asarray(s, np.float64)
        if order == "ascending":
            s = s[np.argsort(s, kind="stable")]
        elif order == "descending":
            s = s[np.argsort(-s, kind="stable")]
        else:
            s = rng.permutation(s)
        cls, pred = labels(rng, len(s))
        check_one_group(ctx, s, cls, pred, rng, f"{name} ({order})")
        check_one_group(ctx, s, np.ones(len(s), np.uint8), pred, rng, f"{name} ({order}, all true)")
        check_one_group(ctx, s, np.zeros(len(s), np.uint8), pred, rng, f"{name} ({order}, all false)")


@pytest.mark.parametrize("kat", SIGNED_ZERO_KATS, ids=lambda k: str(k[0][:6]))
def test_signed_zero_thresholds_known_answers(ctx, kat):
    scores, truth, want = kat
    s, t = np.array(scores, np.float64), np.array(truth, bool)
    n = len(s)
    res = ctx.run(s, np.ones(n), t.astype(np.uint8), np.zeros(n), np.zeros(n), group=np.zeros(n, np.int8))
    assert res["curve_len"][0] == len(want)
    assert_bits_equal(ctx.curve(0, len(want))[2], want, "thresholds")
    res = ctx.run(s, np.ones(n), t.astype(np.uint8), np.zeros(n), np.zeros(n))  # derived groups: a non-indel is a SNP
    assert_bits_equal(ctx.curve(0, int(res["curve_len"][0]))[2], want, "thresholds (SNP)")


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: c[0])
def test_edge_frames_match_the_reference_golden_bit_for_bit(ctx, case):
    name, df, classify_col, group_col = case
    check_against_golden(lambda d: PC.calc_accuracy_metrics(d, classify_col, None, group_col, ctx=ctx),
                         lambda d: PC.calc_recall_precision_curve(d, classify_col, None, group_col, ctx=ctx),
                         df, load_golden()[name])


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_get_concordance_metrics_raises_on_non_finite_scores_like_the_reference(ctx, bad):
    from oracle import concordance_ref as CR

    n = 500
    rng = np.random.default_rng(9)
    scores = np.round(rng.normal(5, 2, n), 1)
    truth, fn_mask = (rng.random(n) < 0.6).astype(int), rng.random(n) < 0.05
    truth[fn_mask] = 1
    pred = (scores > 4).astype(int)
    msg = "Input contains NaN." if np.isnan(bad) else "Input contains infinity or a value too large for dtype('float64')."
    s = scores.copy()
    s[np.flatnonzero(~fn_mask)[7]] = bad
    for kw in ({}, {"return_curves": False}, {"return_metrics": False}):
        with pytest.raises(ValueError) as err:
            PC.get_concordance_metrics(pred, s, truth, fn_mask, ctx=ctx, **kw)
        assert str(err.value) == msg
    with pytest.raises(ValueError) as err:
        CR.concordance_metrics(pred, s, truth, fn_mask)
    assert str(err.value) == msg
    s = scores.copy()
    s[fn_mask] = bad  # false negatives are dropped before sklearn sees the scores
    m, c = PC.get_concordance_metrics(pred, s, truth, fn_mask, ctx=ctx)
    wm, wc = CR.concordance_metrics(pred, s, truth, fn_mask)
    for k in ("precision", "recall", "f1", "predictions"):
        assert_bits_equal(np.asarray(c[k][0], np.float64), wc[k], k)
    s = scores.copy()
    s[np.flatnonzero(~fn_mask)[[3, 9]]] = [np.inf, np.nan]  # NaN's message wins within a selection
    with pytest.raises(ValueError, match="^Input contains NaN.$"):
        PC.get_concordance_metrics(pred, s, truth, fn_mask, ctx=ctx)


def test_more_than_2_24_calls_in_one_group_count_and_divide_exactly(ctx):
    n = (1 << 24) + (1 << 20) + 7
    rng = np.random.default_rng(24)
    cls = (rng.random(n) < 0.97).astype(np.uint8)  # every record called: fp or tp, more than 2^24 of them true
    pred = (rng.random(n) < 0.5).astype(np.uint8)
    zeros8, zeros32 = np.zeros(n, np.uint8), np.zeros(n, np.int32)
    t = cls == 1
    for kind in ("distinct", "tied"):
        s = rng.permutation(n).astype(np.float64) if kind == "distinct" else rng.integers(0, 1000, n).astype(np.float64)
        res = ctx.run(s, pred, cls, zeros8, zeros32)  # non-indels: SNP, derived on the device
        want = np.zeros((9, 8), np.int64)
        want[0] = expected_counts(s, pred, cls, np.ones(n, bool))
        check_counts(res, want, kind)
        assert res["counts"][0, 4] > (1 << 24)
        p, r, thr, tps, fps = exact_curve(s, t)
        d = len(thr)
        assert res["curve_len"][0] == d, kind
        gp, gr, gt = ctx.curve(0, d)
        assert_bits_equal(gp, p, f"{kind}: precision")
        assert_bits_equal(gr, r, f"{kind}: recall")
        assert_bits_equal(gt, thr, f"{kind}: thresholds")
        # the tail (lowest thresholds) is where the counts pass 2^24
        assert tps[-1] > (1 << 24) and gr[0] == 1.0
        for i in (d - 1, d - 2, d // 2):
            o = d - 1 - i
            assert_bits_equal(gp[o], float(Fraction(int(tps[i]), int(tps[i] + fps[i]))), f"{kind}: precision at {i}")
            assert_bits_equal(gr[o], float(Fraction(int(tps[i]), int(tps[-1]))), f"{kind}: recall at {i}")


def _device_run(ctx, cols, group, want_curves=1):
    """ugvc_conc_run on torch CUDA tensors (inputs_on_device = 1) -> the same dict as ConcordanceContext.run."""
    import torch

    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in cols]
    dg = None if group is None else torch.from_numpy(np.ascontiguousarray(group, np.int8)).cuda()
    counts = np.zeros((9, 8), np.int64)
    clen, cut, sel = np.zeros(9, np.int64), np.zeros(9), np.zeros((9, 2), np.int64)
    p = lib._ptr  # noqa: SLF001
    rc = ctx.lib.ugvc_conc_run(ctx.h, len(cols[0]), *(x.data_ptr() for x in d), None if dg is None else dg.data_ptr(), 1,
                               want_curves, p(counts), p(clen), p(cut), p(sel))
    torch.cuda.synchronize()
    assert rc == 0, ctx.lib.ugvc_conc_last_error(ctx.h)
    return {"counts": counts[:, :6], "non_finite": counts[:, 6:], "curve_len": clen, "cutoff": cut, "selected": sel}


def _all_curves(ctx, res):
    return {g: ctx.curve(g, int(res["curve_len"][g])) for g in range(8) if res["curve_len"][g]}


@pytest.mark.parametrize("with_group", [False, True])
def test_inputs_on_device_match_the_host_array_run(ctx, with_group):
    rng = np.random.default_rng(31)
    n = 200_000
    scores = np.round(rng.normal(0, 10, n), 2)
    cls, pred = labels(rng, n)
    indel = (rng.random(n) < 0.3).astype(np.uint8)
    hmer = np.where(indel == 1, rng.integers(-1, 16, n), 0).astype(np.int32)
    group = rng.integers(-1, 7, n).astype(np.int8) if with_group else None
    host = ctx.run(scores, pred, cls, indel, hmer, group=group)
    host_curves = _all_curves(ctx, host)
    assert len(host_curves) >= 2
    dev = _device_run(ctx, (scores, pred, cls, indel, hmer), group)
    for k in ("counts", "non_finite", "curve_len", "selected"):
        np.testing.assert_array_equal(dev[k], host[k], err_msg=k)
    assert_bits_equal(dev["cutoff"], host["cutoff"], "cutoff")
    dev_curves = _all_curves(ctx, dev)
    assert dev_curves.keys() == host_curves.keys()
    for g, hc in host_curves.items():
        for a, b, what in zip(dev_curves[g], hc, ("precision", "recall", "thresholds")):
            assert_bits_equal(a, b, f"{what} of group {g}")


def _curve_rc(ctx, g, capacity):
    out = np.empty(max(1, capacity), np.float64)
    p = lib._ptr(out)  # noqa: SLF001
    return ctx.lib.ugvc_conc_curve(ctx.h, g, p, p, p, capacity)


def test_handle_reuse_and_curve_refusals(ctx):
    rng = np.random.default_rng(41)
    n = 5000
    scores = np.round(rng.normal(3, 2, n), 1)
    cls, pred = labels(rng, n)
    indel = (rng.random(n) < 0.4).astype(np.uint8)
    hmer = np.where(indel == 1, rng.integers(0, 14, n), 0).astype(np.int32)
    res = ctx.run(scores, pred, cls, indel, hmer)
    d = int(res["curve_len"][0])
    assert d > 1
    assert _curve_rc(ctx, 0, d - 1) == lib.UGVC_E_ARG  # capacity too small
    for g in (-1, 9, 100):
        assert _curve_rc(ctx, g, d) == lib.UGVC_E_ARG
    assert _curve_rc(ctx, 0, d) == 0
    # a metrics-only run on the same handle drops the curves of the run before
    res2 = ctx.run(scores, pred, cls, indel, hmer, want_curves=False)
    check_counts(res2, np.hstack([res["counts"], res["non_finite"]]), "metrics-only run")
    assert not res2["curve_len"].any()
    for g in range(9):
        assert _curve_rc(ctx, g, 0) == 0  # nothing left to copy, so no capacity is too small
    # two contexts stay independent
    other = PC.ConcordanceContext(0)
    try:
        a = ctx.run(scores, pred, cls, indel, hmer)
        cls_b = np.where(cls == 1, 0, 1).astype(np.uint8)
        b = other.run(-scores, pred, cls_b, indel, hmer)
        for c, r, s_, k_, who in ((ctx, a, scores, cls, "first"), (other, b, -scores, cls_b, "second")):
            for g in range(8):
                sel = _members(indel, hmer, g) & (k_ != 2)
                assert r["curve_len"][g] > 0, g
                for x, y, what in zip(c.curve(g, int(r["curve_len"][g])), exact_curve(s_[sel], k_[sel] == 1)[:3],
                                      ("precision", "recall", "thresholds")):
                    assert_bits_equal(x, y, f"{what} of group {g} on the {who} context")
    finally:
        other.close()


def _members(indel, hmer, g):
    if g == 7:
        return indel == 1
    gid = np.full(len(indel), -1)
    gid[indel == 0] = 0
    gid[(indel == 1) & (hmer == 0)] = 1
    for k, lo, hi in ((2, 1, 4), (3, 5, 7), (4, 8, 10), (5, 11, 12), (6, 13, 1 << 30)):
        gid[(indel == 1) & (hmer >= lo) & (hmer <= hi)] = k
    return gid == g


@pytest.mark.parametrize("bad", [("group", v) for v in (7, 8, 9, 15, 127, -2, -128)] + [("cls", v) for v in (4, 255)],
                         ids=lambda b: f"{b[0]}={b[1]}")
def test_ids_outside_the_abi_are_refused_and_count_nothing(ctx, bad):
    rng = np.random.default_rng(51)
    n = 70_000
    scores = rng.random(n)
    cls, pred = labels(rng, n)
    group = rng.integers(-1, 7, n).astype(np.int8)
    col, v = bad
    for at in (0, n // 2, n - 1):
        g, c = group.copy(), cls.copy()
        if col == "group":
            g[at] = np.int8(v)
        else:
            c[at] = np.uint8(v)
        counts = np.full((9, 8), -1, np.int64)
        clen, cut, sel = np.full(9, -1, np.int64), np.full(9, -1.0), np.full((9, 2), -1, np.int64)
        p = lib._ptr  # noqa: SLF001
        rc = ctx.lib.ugvc_conc_run(ctx.h, n, p(scores), p(pred), p(c), p(np.zeros(n, np.uint8)), p(np.zeros(n, np.int32)),
                                   p(g), 0, 1, p(counts), p(clen), p(cut), p(sel))
        assert rc == lib.UGVC_E_ARG, ctx.lib.ugvc_conc_last_error(ctx.h)
        assert not counts.any() and not clen.any() and not cut.any() and not sel.any()
        for gg in range(9):
            assert _curve_rc(ctx, gg, 0) == 0
    # the handle still works
    res = ctx.run(scores, pred, cls, np.zeros(n), np.zeros(n), group=group)
    for gg in range(7):
        want = expected_counts(scores, pred, cls, group == gg)
        np.testing.assert_array_equal(res["counts"][gg], want[:6])
        np.testing.assert_array_equal(res["non_finite"][gg], want[6:])
