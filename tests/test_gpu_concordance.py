"""GPU: the concordance metrics of BASELINE configs[4] (variantcalling_b200.concordance over
csrc/concordance.cu) against the reference's own outputs (golden) and, at a larger size, the
oracle restatement: counts equal, precision / recall / F1 curves bit-identical."""
import numpy as np
import pytest

from oracle import concordance_ref as CR
from tests.concordance_data import make_cases, make_frame
from tests.test_concordance_cpu import assert_bits_equal, check_accuracy, check_curve, load_golden
from variantcalling_b200 import concordance as PC

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", list(make_cases()), ids=lambda c: c[0])
def test_metrics_and_curves_match_the_reference_golden(case):
    name, df, classify_col, group_col = case
    want = load_golden()[name]
    check_accuracy(PC.calc_accuracy_metrics(df.copy(), classify_col, None, group_col), want["accuracy"])
    check_curve(PC.calc_recall_precision_curve(df.copy(), classify_col, None, group_col), want["curve"])


def test_two_million_records_against_the_oracle():
    df = make_frame(2_000_000, 99)
    ctx = PC.ConcordanceContext(0)
    acc = PC.calc_accuracy_metrics(df.copy(), "classify_gt", ctx=ctx)
    curve = PC.calc_recall_precision_curve(df.copy(), "classify_gt", ctx=ctx)
    assert ctx.launch_count() > 10
    want_acc, want_curve = CR.calc_accuracy_metrics(df, "classify_gt"), CR.calc_recall_precision_curve(df, "classify_gt")
    for col in CR.METRIC_COLUMNS:
        np.testing.assert_array_equal(acc[col].to_numpy(dtype=np.float64), want_acc[col].to_numpy(dtype=np.float64), err_msg=col)
    for col in ("precision", "recall", "f1", "predictions"):
        for g, got, exp in zip(want_curve["group"], curve[col], want_curve[col]):
            np.testing.assert_array_equal(np.asarray(got), np.asarray(exp), err_msg=f"{col} of {g}")
    assert list(curve["threshold"]) == list(want_curve["threshold"])
    # size-independent properties: recall never increases with the threshold, counts add up
    snp = curve.iloc[0]
    assert np.all(np.diff(snp["recall"]) <= 0) and np.all(np.diff(snp["predictions"]) > 0)
    assert int(acc["initial_tp"][:7].sum() + acc["initial_fp"][:7].sum() + acc["initial_fn"][:7].sum()) == len(df)


def test_get_concordance_metrics_single_selection():
    rng = np.random.default_rng(3)
    n = 5000
    truth = (rng.random(n) < 0.7).astype(int)
    scores = np.round(rng.normal(np.where(truth, 5, 3), 2), 1)
    fn_mask = rng.random(n) < 0.05
    truth[fn_mask] = 1
    pred = (scores > 3.5).astype(int)
    m, c = PC.get_concordance_metrics(pred, scores, truth, fn_mask)
    wm, wc = CR.concordance_metrics(pred, scores, truth, fn_mask)
    for k in CR.METRIC_COLUMNS:
        assert m[k][0] == wm[k], k
    for k in ("precision", "recall", "f1", "predictions"):
        np.testing.assert_array_equal(np.asarray(c[k][0]), wc[k])
    assert c["threshold"][0] == wc["threshold"]


def test_evaluate_concordance_cli_writes_the_reference_csvs(tmp_path):
    """`python ugvc evaluate_concordance`: .stats.csv / .thresholds.csv as evaluate_concordance.py:100-107 writes them."""
    import pandas as pd

    from variantcalling_b200 import evaluate_concordance as EC

    df = make_frame(30000, 42)
    src = str(tmp_path / "cmp.csv")
    df.to_csv(src, index=False)
    prefix = str(tmp_path / "out")
    EC.run(["--input_file", src, "--output_prefix", prefix])
    # the outputs hold shortest round-trip reprs: read them back exactly and compare bit for bit (the input is read
    # as the CLI reads it)
    stats = pd.read_csv(prefix + ".stats.csv", sep=";", float_precision="round_trip")
    want = CR.calc_accuracy_metrics(pd.read_csv(src), "classify_gt")
    assert list(stats.columns) == ["group"] + CR.METRIC_COLUMNS and list(stats["group"]) == list(want["group"])
    for col in CR.METRIC_COLUMNS:
        assert_bits_equal(stats[col].to_numpy(dtype=float), want[col].to_numpy(dtype=float), col)
    thr = pd.read_csv(prefix + ".thresholds.csv", float_precision="round_trip")
    want_thr = CR.calc_recall_precision_curve(pd.read_csv(src), "classify_gt")
    assert list(thr["group"]) == list(want_thr["group"])
    assert_bits_equal(thr["threshold"].to_numpy(dtype=float), np.asarray(list(want_thr["threshold"]), dtype=float), "threshold")
