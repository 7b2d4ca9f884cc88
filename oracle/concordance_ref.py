"""ORACLE (test infrastructure, not product code): precision / recall of a filtered call set
against truth -- BASELINE.json configs[4], the caller-side step after filter_variants_pipeline.

CPU restatement (NumPy / pandas) of
  * ``calc_accuracy_metrics``          ugbio_core/concordance/concordance_utils.py:11-106
  * ``calc_recall_precision_curve``    :109-188
  * ``validate_preprocess_concordance`` :191-225, ``convert_filter2call`` :228-243,
    ``get_selection_functions`` / ``add_grouping_column`` :266-300
  * ``get_concordance_metrics``        :346-458
  * ``precision_recall_curve`` / ``get_precision`` / ``get_recall`` / ``get_f1``
                                       ugbio_core/stats_utils.py:76-210
  * the third-party ``sklearn.metrics.precision_recall_curve`` the latter calls (scikit-learn,
    reference pin 1.5.x; published algorithm: stable sort by decreasing score, cumulative true /
    false positives at each distinct score, precision = tps / (tps + fps), recall = tps / tps[-1],
    reversed, with a final (1, 0) point).

PARITY STATUS: pinned -- tests/golden/concordance_metrics.json.gz holds the output of the
reference's own functions (scripts/make_golden_concordance.py imports them from /root/reference)
on the frames of tests/concordance_data.py; tests/test_concordance_cpu.py compares.
"""
from __future__ import annotations

import numpy as np
import pandas as pd

GROUPS = ["SNP", "Non-hmer INDEL", "HMER indel <= 4", "HMER indel (4,8)", "HMER indel [8,10]", "HMER indel 11,12",
          "HMER indel > 12"]
METRIC_COLUMNS = ["tp", "fp", "fn", "precision", "recall", "f1", "initial_tp", "initial_fp", "initial_fn",
                  "initial_precision", "initial_recall", "initial_f1"]


def default_group(indel: np.ndarray, hmer: np.ndarray) -> np.ndarray:
    """Group name per record (object array, None when no selection function matches), :266-300."""
    out = np.full(indel.shape, None, dtype=object)
    out[~indel] = GROUPS[0]
    out[indel & (hmer == 0)] = GROUPS[1]
    for name, lo, hi in ((GROUPS[2], 1, 4), (GROUPS[3], 5, 7), (GROUPS[4], 8, 10), (GROUPS[5], 11, 12)):
        out[indel & (hmer >= lo) & (hmer <= hi)] = name
    out[indel & (hmer > 12)] = GROUPS[6]  # noqa: PLR2004
    return out


def assert_all_finite(y_score: np.ndarray):
    """sklearn.utils.assert_all_finite as _binary_clf_curve calls it: NaN's message before inf's."""
    if y_score.dtype.kind != "f":
        return
    if np.isnan(y_score).any():
        raise ValueError("Input contains NaN.")
    if np.isinf(y_score).any():
        raise ValueError(f"Input contains infinity or a value too large for {y_score.dtype!r}.")


def sklearn_pr_curve(y_true: np.ndarray, y_score: np.ndarray):
    """A run of equal scores reports its first score in input order (the stable ascending sort, reversed, keeps
    the run's last index, which is its first in input order): a run of -0.0 and +0.0 keeps its first zero's sign."""
    assert_all_finite(y_score)
    order = np.argsort(y_score, kind="mergesort")[::-1]
    y_score, y_true = y_score[order], y_true[order]
    idx = np.r_[np.where(np.diff(y_score))[0], y_true.size - 1]
    tps = np.cumsum(y_true, dtype=np.float64)[idx]
    fps = 1 + idx - tps
    ps = tps + fps
    precision = np.zeros_like(tps)
    np.divide(tps, ps, out=precision, where=(ps != 0))
    recall = np.ones_like(tps) if tps[-1] == 0 else tps / tps[-1]
    return np.hstack((precision[::-1], 1)), np.hstack((recall[::-1], 0)), y_score[idx][::-1]


def pr_curve_with_fn(truth: np.ndarray, scores: np.ndarray, fn_mask: np.ndarray, min_count: int = 20):
    """stats_utils.precision_recall_curve (pos_label=1): -> precisions, recalls, f1, thresholds"""
    if len(truth) == 0:
        e = np.array([])
        return e, e, e, e
    assert len(set(truth)) <= 2, "Only up to two classes of variant labels are possible"  # noqa: S101, PLR2004
    sel_truth = truth[~fn_mask] == 1
    sel_scores = scores[~fn_mask]
    n_fn = fn_mask.sum()
    if len(sel_truth) > 0:
        raw_p, raw_r, thr = sklearn_pr_curve(sel_truth, sel_scores)
    else:
        with np.errstate(all="ignore"):
            raw_p = np.array([sel_truth.sum() / len(sel_truth), 1.0])
        raw_r = np.array([1.0, 0.0])
        thr = np.array([0])
    with np.errstate(all="ignore"):
        correction = sel_truth.sum() / (sel_truth.sum() + n_fn)
    recalls = (raw_r * correction)[1:-1]
    precisions = raw_p[1:-1]
    thr = thr[1:]
    f1 = 2 * (recalls * precisions) / (recalls + precisions + np.finfo(float).eps)
    ordered = np.sort(sel_scores)
    cutoff = ordered[max(0, len(ordered) - min_count)] if len(ordered) > 0 else 0
    keep = ~(thr > cutoff)
    return precisions[keep], recalls[keep], f1[keep], thr[keep]


def _ratio_complement(bad, good):  # get_precision / get_recall: 1 when nothing was counted
    return 1 if bad + good == 0 else 1 - bad / (bad + good)


def _f1(p, r):
    if np.nan in {p, r}:
        return np.nan
    return 0 if p + r == 0 else 2 * p * r / (p + r)


def concordance_metrics(pred: np.ndarray, scores: np.ndarray, truth: np.ndarray, fn_mask: np.ndarray):
    """-> (metrics dict, curve dict), get_concordance_metrics :346-458"""
    p, r, f1, thr = pr_curve_with_fn(truth, scores, fn_mask)
    threshold = thr[np.argmax(f1)] if len(f1) > 0 else 0
    curve = {"predictions": thr, "precision": p, "recall": r, "f1": f1, "threshold": threshold}
    n_fn = fn_mask.sum()
    pred, truth = pred[~fn_mask], truth[~fn_mask]
    if len(pred) == 0:
        m = dict.fromkeys(METRIC_COLUMNS, 1.0)
        for k in ("tp", "fp", "fn", "initial_tp", "initial_fp", "initial_fn"):
            m[k] = 0
        return m, {"threshold": 0, "predictions": [], "precision": [], "recall": [], "f1": []}
    tp = ((truth > 0) & (pred > 0) & (truth == pred)).sum()
    fp = (pred > truth).sum()
    fn = n_fn + (pred < truth).sum()
    itp = (truth > 0).sum()
    ifp = len(truth) - itp
    prec, rec = _ratio_complement(fp, tp), _ratio_complement(fn, tp)
    iprec, irec = _ratio_complement(ifp, itp), _ratio_complement(n_fn, itp)
    return ({"tp": tp, "fp": fp, "fn": fn, "precision": prec, "recall": rec, "f1": _f1(prec, rec), "initial_tp": itp,
             "initial_fp": ifp, "initial_fn": n_fn, "initial_precision": iprec, "initial_recall": irec,
             "initial_f1": _f1(iprec, irec)}, curve)


def _prepared(df: pd.DataFrame, group_col):
    """validate_preprocess_concordance + vc_call + grouping: -> (frame, group labels)"""
    assert "tree_score" in df.columns, "Input concordance file should be after applying a model"  # noqa: S101
    df = df.copy()
    df.loc[pd.isna(df["filter"]), "filter"] = "PASS"
    df.loc[pd.isna(df["tree_score"]), "tree_score"] = 0
    if group_col is not None:
        df = df[~pd.isna(df[group_col])]
        labels = df[group_col].to_numpy()
    else:
        labels = default_group(df["indel"].to_numpy(dtype=bool), df["hmer_indel_length"].to_numpy())
    # convert_filter2call resets its ignored_filters argument to {"PASS"} (:242): only PASS passes
    df["vc_call"] = [1 if all(f == "PASS" for f in s.split(";")) else 0 for s in df["filter"]]
    return df, labels


def _per_group(df, labels, classify_col, want):
    truth_code = df[classify_col].map({"tp": 1, "fn": 1, "fp": 0, "tn": 0}).to_numpy()
    fn_mask = (df[classify_col] == "fn").to_numpy()
    pred, scores = df["vc_call"].to_numpy(), df["tree_score"].to_numpy(dtype=np.float64)
    selections = [(g, labels == g) for g in GROUPS] + [("INDELS", df["indel"].to_numpy(dtype=bool))]
    if want == "metrics":
        selections.append(("H-INDELS", df["hmer_indel_length"].to_numpy() > 0))
    for name, sel in selections:
        yield name, concordance_metrics(pred[sel], scores[sel], truth_code[sel], fn_mask[sel])


def calc_accuracy_metrics(df, classify_col, group_col=None) -> pd.DataFrame:
    frame, labels = _prepared(df, group_col)
    rows = []
    for name, (m, _curve) in _per_group(frame, labels, classify_col, "metrics"):
        rows.append({"group": name, **m})
    out = pd.DataFrame(rows, columns=["group"] + METRIC_COLUMNS)
    return out.round(5)


def calc_recall_precision_curve(df, classify_col, group_col=None) -> pd.DataFrame:
    frame, labels = _prepared(df, group_col)
    rows = []
    for name, (_m, c) in _per_group(frame, labels, classify_col, "curve"):
        rows.append({"group": name, "precision": c["precision"], "recall": c["recall"], "f1": c["f1"],
                     "threshold": c["threshold"], "predictions": c["predictions"]})
    return pd.DataFrame(rows, columns=["group", "precision", "recall", "f1", "threshold", "predictions"])
