"""CPU: the oracle's restatement of evaluate_concordance's metrics against the reference's own
functions (tests/golden/concordance_metrics.json.gz, scripts/make_golden_concordance.py)."""
import gzip
import json
import os

import numpy as np
import pytest

from oracle import concordance_ref as CR
from tests.concordance_data import make_cases, make_edge_cases, make_error_cases
from variantcalling_b200 import lib

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "concordance_metrics.json.gz")


def load_golden():
    with gzip.open(GOLDEN, "rt") as fh:
        return json.load(fh)


def as_float(values):
    return np.array([np.nan if v is None else v for v in values], dtype=np.float64)


def check_accuracy(acc, want):
    assert list(acc["group"]) == want["group"]
    for col in CR.METRIC_COLUMNS:
        # the reference rounds to 5 decimals in its own (pandas < 3) environment; see the generator's note
        np.testing.assert_array_equal(np.round(acc[col].to_numpy(dtype=np.float64), 5), np.round(as_float(want[col]), 5), err_msg=col)


def check_curve(curve, want):
    assert list(curve["group"]) == want["group"]
    for col in ("precision", "recall", "f1"):
        for g, got, exp in zip(want["group"], curve[col], want[col]):
            np.testing.assert_array_equal(np.asarray(got, dtype=np.float64), as_float(exp), err_msg=f"{col} of {g}")
    np.testing.assert_array_equal(np.asarray(list(curve["threshold"]), dtype=np.float64), as_float(want["threshold"]))


def bits(values) -> np.ndarray:
    """fp64 values as their uint64 bit patterns (every NaN as NumPy's one NaN: JSON keeps no payload)."""
    a = np.asarray(values, dtype=np.float64)
    return np.where(np.isnan(a), np.nan, a).view(np.uint64)


def assert_bits_equal(got, want, what):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape, f"{what}: {g.shape} points, want {w.shape}"
    bad = np.flatnonzero(g != w)
    assert len(bad) == 0, f"{what}: {len(bad)} values differ, first at {bad[0]}: {np.asarray(got, np.float64).ravel()[bad[0]]!r} " \
                          f"want {np.asarray(want, np.float64).ravel()[bad[0]]!r}"


def check_accuracy_bits(acc, want):
    """Counts exact; ratios rounded to 5 decimals (the reference's own environment rounds) and compared bit for bit."""
    assert list(acc["group"]) == want["group"]
    for col in CR.METRIC_COLUMNS:
        assert_bits_equal(np.round(acc[col].to_numpy(dtype=np.float64), 5), np.round(as_float(want[col]), 5), col)


def check_curve_bits(curve, want):
    assert list(curve["group"]) == want["group"]
    for col in ("precision", "recall", "f1", "predictions"):
        for g, got, exp in zip(want["group"], curve[col], want[col]):
            assert_bits_equal(np.asarray(got, dtype=np.float64), as_float(exp), f"{col} of {g}")
    assert_bits_equal(np.asarray(list(curve["threshold"]), dtype=np.float64), as_float(want["threshold"]), "threshold")


def check_against_golden(accuracy_fn, curve_fn, df, want):
    """accuracy_fn / curve_fn: frame -> frame.  Where the reference raised, the same type and message."""
    for key, fn, check in (("accuracy", accuracy_fn, check_accuracy_bits), ("curve", curve_fn, check_curve_bits)):
        if "error" in want[key]:
            with pytest.raises(Exception) as err:  # noqa: PT011
                fn(df.copy())
            assert [type(err.value).__name__, str(err.value)] == want[key]["error"], key
        else:
            check(fn(df.copy()), want[key])


EDGE_CASES = list(make_edge_cases()) + list(make_error_cases())

# A run of equal scores reports its first score in input order: with signed zeros, its first zero's sign.
# (scores, truth) -> the raw curve's thresholds in increasing order, derived by hand.
SIGNED_ZERO_KATS = [
    ([-0.0, 0.0, 0.0, 1.0, 2.0, 0.0] * 5, [1, 0, 1, 0, 1, 1] * 5, [-0.0, 1.0, 2.0]),
    ([0.0, -0.0, -0.0, 1.0], [1, 0, 1, 1], [0.0, 1.0]),
    ([1.0, -0.0, 0.0], [0, 1, 0], [-0.0, 1.0]),
    ([-0.0, -3.0, 0.0, -3.0], [0, 1, 1, 0], [-3.0, -0.0]),
    ([0.0], [1], [0.0]),
    ([-0.0], [0], [-0.0]),
    ([5.0, -0.0, 5.0, 0.0, -0.0], [1, 1, 0, 0, 1], [-0.0, 5.0]),
]


@pytest.mark.parametrize("case", list(make_cases()), ids=lambda c: c[0])
def test_oracle_reproduces_the_reference(case):
    name, df, classify_col, group_col = case
    want = load_golden()[name]
    check_accuracy(CR.calc_accuracy_metrics(df, classify_col, group_col), want["accuracy"])
    check_curve(CR.calc_recall_precision_curve(df, classify_col, group_col), want["curve"])


class DeviceModel:
    """NumPy model of what csrc/concordance.cu returns (the ugvc_conc_run / ugvc_conc_curve contract of
    include/ugvc_b200.h), so that the host mirror's arithmetic is covered without a GPU."""

    def run(self, scores, pred, cls, indel, hmer, group=None, want_curves=True):
        scores, pred, cls = np.asarray(scores, np.float64), np.asarray(pred).astype(bool), np.asarray(cls)
        indel, hmer = np.asarray(indel).astype(bool), np.asarray(hmer)
        if (cls > 3).any() or (group is not None and ((np.asarray(group) < -1) | (np.asarray(group) > 6)).any()):  # noqa: PLR2004
            raise lib.UgvcError(lib.UGVC_E_ARG, "conc_run: a group id outside -1..6 or a class code above 3")
        if group is None:
            gid = np.full(len(cls), -1)
            gid[~indel] = 0
            gid[indel & (hmer == 0)] = 1
            for g, lo, hi in ((2, 1, 4), (3, 5, 7), (4, 8, 10), (5, 11, 12), (6, 13, 1 << 30)):
                gid[indel & (hmer >= lo) & (hmer <= hi)] = g
        else:
            gid = np.asarray(group)
        truth, fnm = (cls == 1) | (cls == 2), cls == 2
        members = [gid == g for g in range(7)] + [indel, hmer > 0]
        counts, non_finite = np.zeros((9, 6), np.int64), np.zeros((9, 2), np.int64)
        self.curves, curve_len, cutoff, selected = {}, np.zeros(9, np.int64), np.zeros(9), np.zeros((9, 2), np.int64)
        for g, m in enumerate(members):
            called = m & ~fnm
            t, p = truth[called], pred[called]
            s = scores[called]
            counts[g] = [(t & p).sum(), (p & ~t).sum(), (~p & t).sum(), t.sum(), called.sum(), (m & fnm).sum()]
            non_finite[g] = [np.isnan(s).sum(), np.isinf(s).sum()]
            # the device draws a curve over non-finite scores too; the host raises before it reads one
            if want_curves and g < 8 and called.any() and np.isfinite(s).all():
                raw_p, raw_r, thr = CR.sklearn_pr_curve(t, scores[called])
                self.curves[g] = (raw_p[:-1], raw_r[:-1], thr)
                curve_len[g] = len(thr)
                cutoff[g] = np.sort(scores[called])[::-1][min(called.sum() - 1, 19)]
                selected[g] = [called.sum(), t.sum()]
        return {"counts": counts, "non_finite": non_finite, "curve_len": curve_len, "cutoff": cutoff, "selected": selected}

    def curve(self, g, n):
        return self.curves[g]


@pytest.mark.parametrize("case", list(make_cases()), ids=lambda c: c[0])
def test_host_mirror_arithmetic_on_a_device_model(case):
    from variantcalling_b200 import concordance as PC

    name, df, classify_col, group_col = case
    want = load_golden()[name]
    check_accuracy(PC.calc_accuracy_metrics(df.copy(), classify_col, None, group_col, ctx=DeviceModel()), want["accuracy"])
    check_curve(PC.calc_recall_precision_curve(df.copy(), classify_col, None, group_col, ctx=DeviceModel()), want["curve"])


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: c[0])
def test_oracle_reproduces_the_reference_at_the_edges(case):
    name, df, classify_col, group_col = case
    check_against_golden(lambda d: CR.calc_accuracy_metrics(d, classify_col, group_col),
                         lambda d: CR.calc_recall_precision_curve(d, classify_col, group_col), df, load_golden()[name])


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: c[0])
def test_host_mirror_on_a_device_model_at_the_edges(case):
    from variantcalling_b200 import concordance as PC

    name, df, classify_col, group_col = case
    check_against_golden(lambda d: PC.calc_accuracy_metrics(d, classify_col, None, group_col, ctx=DeviceModel()),
                         lambda d: PC.calc_recall_precision_curve(d, classify_col, None, group_col, ctx=DeviceModel()),
                         df, load_golden()[name])


def test_golden_records_the_scikit_learn_version_and_no_signed_zero():
    assert load_golden()["_meta"]["sklearn"]
    for name, df, _c, _g in EDGE_CASES:  # scikit-learn after 1.5 gives a tie run of zeros another sign (see the generator)
        s = df["tree_score"].to_numpy(dtype=np.float64)
        assert not np.any((s == 0) & np.signbit(s)), name


@pytest.mark.parametrize("kat", SIGNED_ZERO_KATS, ids=lambda k: str(k[0][:6]))
def test_oracle_signed_zero_thresholds(kat):
    scores, truth, want = kat
    for order in (slice(None), slice(None, None, -1)):  # the rule holds whatever the input order
        s, t = np.array(scores)[order], np.array(truth, bool)[order]
        thr = CR.sklearn_pr_curve(t, s)[2]
        first = [s[np.flatnonzero(s == v)[0]] for v in thr]  # the first score of each run, in input order
        assert_bits_equal(thr, first, "thresholds")
        if order == slice(None):
            assert_bits_equal(thr, want, "thresholds")


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_get_concordance_metrics_non_finite_on_a_device_model(bad):
    from variantcalling_b200 import concordance as PC

    n = 60
    scores, truth, fn_mask = np.arange(n, dtype=np.float64), np.arange(n) % 3 != 0, np.arange(n) % 7 == 0
    pred = (scores > 20).astype(int)
    msg = "Input contains NaN." if np.isnan(bad) else "Input contains infinity or a value too large for dtype('float64')."
    for where, raises in ((np.flatnonzero(~fn_mask)[4], True), (np.flatnonzero(fn_mask)[2], False)):
        s = scores.copy()
        s[where] = bad
        for kw in ({}, {"return_curves": False}, {"return_metrics": False}):
            if raises:
                for fn in (lambda: PC.get_concordance_metrics(pred, s, truth, fn_mask, ctx=DeviceModel(), **kw),
                           lambda: CR.concordance_metrics(pred, s, truth, fn_mask)):
                    with pytest.raises(ValueError) as err:
                        fn()
                    assert str(err.value) == msg
            else:
                PC.get_concordance_metrics(pred, s, truth, fn_mask, ctx=DeviceModel(), **kw)
                CR.concordance_metrics(pred, s, truth, fn_mask)
    s = scores.copy()
    s[[3, 5]] = [np.inf, np.nan]  # within one selection NaN's message wins
    with pytest.raises(ValueError, match="^Input contains NaN.$"):
        PC.get_concordance_metrics(pred, s, truth, fn_mask, ctx=DeviceModel())
    with pytest.raises(ValueError, match="^Input contains NaN.$"):
        CR.concordance_metrics(pred, s, truth, fn_mask)


def test_non_finite_message_of_the_first_group_in_the_reference_order():
    from variantcalling_b200 import concordance as PC

    raise_ = PC._raise_on_non_finite  # noqa: SLF001
    called = np.array([1.0, np.inf, np.nan])
    nf = np.zeros((9, 2), np.int64)
    nf[5, 0] = 1  # NaN in HMER indel 11,12
    nf[2, 1] = 4  # inf in HMER indel <= 4: the reference meets it first
    with pytest.raises(ValueError, match="infinity"):
        raise_(called, {"non_finite": nf}, range(9), np.dtype(np.float64))
    nf[2, 1] = 0
    nf[8, 1] = 1  # H-INDELS only: the metrics raise, the curves do not
    with pytest.raises(ValueError, match="NaN"):
        raise_(called, {"non_finite": nf}, range(9), np.dtype(np.float64))
    nf[5, 0] = 0
    raise_(called, {"non_finite": nf}, range(8), np.dtype(np.float64))
    with pytest.raises(ValueError, match=r"dtype\('float32'\)"):
        raise_(called, {"non_finite": nf}, range(9), np.dtype(np.float32))
    raise_(np.array([0.0, -1e308]), {}, range(9), np.dtype(np.float64))  # all finite: nothing to look up


@pytest.mark.parametrize("bad", [{"group": 7}, {"group": 9}, {"group": -2}, {"group": 127}, {"cls": 4}, {"cls": 255}])
def test_device_model_refuses_ids_outside_the_abi(bad):
    n = 10
    cols = {"cls": np.ones(n, np.uint8), "group": np.zeros(n, np.int8)}
    k, v = next(iter(bad.items()))
    cols[k] = cols[k].astype(np.int64)
    cols[k][4] = v
    with pytest.raises(lib.UgvcError) as err:
        DeviceModel().run(np.arange(n, dtype=np.float64), np.ones(n), cols["cls"], np.zeros(n), np.zeros(n), cols["group"])
    assert err.value.code == lib.UGVC_E_ARG
