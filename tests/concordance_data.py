"""Synthetic concordance frames (the columns evaluate_concordance reads from the comparison HDF5:
``filter``, ``tree_score``, ``classify`` / ``classify_gt``, ``indel``, ``hmer_indel_length``,
``hmer_indel_nuc``), deterministic, shared by the golden generator and the tests."""
from __future__ import annotations

import numpy as np
import pandas as pd


def make_frame(n: int, seed: int, *, p_fn=0.03, score_decimals=None, with_tn=False, nan_scores=0) -> pd.DataFrame:
    rng = np.random.default_rng(seed)
    indel = rng.random(n) < 0.25
    hmer = np.where(indel & (rng.random(n) < 0.7), rng.integers(1, 16, size=n), 0)
    hmer = np.where(~indel & (rng.random(n) < 0.01), rng.integers(1, 5, size=n), hmer)  # hmer length on a non-indel row
    truth = rng.random(n) < 0.8
    # scores: float32 values (TREE_SCORE read back from a VCF), higher for true calls
    score = np.clip(rng.normal(np.where(truth, 60, 25), 18), 0, None).astype(np.float32).astype(np.float64)
    if score_decimals is not None:
        score = np.round(score, score_decimals)  # many ties
    classify = np.where(truth, "tp", "fp").astype(object)
    fn = rng.random(n) < p_fn
    classify[fn] = "fn"
    if with_tn:
        classify[(rng.random(n) < 0.02) & ~fn] = "tn"
    low = score <= 30.0  # noqa: PLR2004
    other = rng.random(n) < 0.04
    filt = np.where(low & other, "LOW_SCORE;HPOL_RUN", np.where(low, "LOW_SCORE", np.where(other, "HPOL_RUN", "PASS"))).astype(object)
    filt[rng.random(n) < 0.01] = "PASS;PASS"
    score[fn] = np.nan if nan_scores else score[fn]
    if nan_scores:
        score[rng.integers(0, n, size=nan_scores)] = np.nan
    # genotype-aware classification differs on a few rows
    classify_gt = classify.copy()
    flip = (rng.random(n) < 0.03) & (classify == "tp")
    classify_gt[flip] = "fp"
    return pd.DataFrame({"filter": filt, "tree_score": score, "classify": classify, "classify_gt": classify_gt,
                         "indel": indel, "hmer_indel_length": hmer.astype(np.int64),
                         "hmer_indel_nuc": np.where(hmer > 0, "A", None)})


def make_cases():
    """(name, frame, classify column, group column or None)"""
    yield "mixed_6k", make_frame(6000, 1), "classify", None
    yield "mixed_gt_ties", make_frame(9000, 2, score_decimals=0), "classify_gt", None
    yield "tiny_groups", make_frame(120, 3, p_fn=0.1), "classify", None           # groups below the 20-call cutoff
    yield "with_tn_and_nan", make_frame(2500, 4, with_tn=True, nan_scores=25), "classify", None
    f = make_frame(2000, 5)
    f.loc[f["indel"], "classify"] = "fn"                                          # every indel group: only false negatives
    yield "all_fn_indels", f, "classify", None
    f = make_frame(2000, 6)
    f = f[~f["indel"]].reset_index(drop=True)                                     # empty indel groups
    yield "snps_only", f, "classify", None
    f = make_frame(3000, 7)
    f["my_group"] = np.where(f["indel"], "Non-hmer INDEL", "SNP")
    f.loc[::17, "my_group"] = None                                                # rows without a type are dropped
    yield "custom_group_column", f, "classify", "my_group"


def _frame(scores, classify, indel=None, hmer=None, filt=None, **extra) -> pd.DataFrame:
    """A frame with the columns the metrics read, from per-record arrays (defaults: SNPs, all PASS)."""
    n = len(scores)
    indel = np.zeros(n, bool) if indel is None else np.asarray(indel, bool)
    hmer = np.zeros(n, np.int64) if hmer is None else np.asarray(hmer)
    filt = np.full(n, "PASS", object) if filt is None else np.asarray(filt, object)
    classify = np.asarray(classify, object)
    nuc = np.where(np.nan_to_num(hmer, nan=0) > 0, "A", None)
    return pd.DataFrame({"filter": filt, "tree_score": np.asarray(scores, np.float64), "classify": classify,
                         "classify_gt": classify.copy(), "indel": indel, "hmer_indel_length": hmer,
                         "hmer_indel_nuc": nuc, **extra})


def _labels(rng, n, p_true=0.7, p_fn=0.05):
    truth = rng.random(n) < p_true
    cls = np.where(truth, "tp", "fp").astype(object)
    cls[rng.random(n) < p_fn] = "fn"
    return cls


def _filters(rng, scores, cut):
    return np.where((scores > cut) | (rng.random(len(scores)) < 0.05), "PASS", "LOW_SCORE").astype(object)


def _round(x, decimals):
    return np.round(x, decimals) + 0.0  # -0.0 + 0.0 is +0.0: no signed zeros in the golden frames


def _spread(rng, values, n):
    """n draws from `values` (each at least once when n allows), shuffled."""
    out = np.concatenate([values, rng.choice(values, size=max(0, n - len(values)))])[:n]
    return rng.permutation(out)


def ulp_family():
    """Scores one ulp apart around a few bases, both signs (no zero)."""
    bases = np.array([1.0, 37.5, -3.25, 1e-300, -1e300, 0.1, 2.0 ** 52])
    vals = np.concatenate([bases, np.nextafter(bases, np.inf), np.nextafter(bases, -np.inf),
                           np.nextafter(np.nextafter(bases, np.inf), np.inf)])
    return vals


def extreme_family():
    """Subnormals, the smallest and largest magnitudes and +-1e308, with +0.0 (never -0.0) and a few normals."""
    tiny = np.nextafter(0.0, 1.0)
    return np.array([tiny, 2 * tiny, -tiny, 2.2250738585072009e-308, -2.2250738585072009e-308, 2.2250738585072014e-308,
                     1e308, -1e308, np.finfo(np.float64).max, -np.finfo(np.float64).max, 0.0, 1.0, -1.0, 12.5])


def make_edge_cases():
    """(name, frame, classify column, group column or None): score families and group edges that the reference's
    own functions score (tests/golden/concordance_metrics.json.gz, next to make_cases)."""
    rng = np.random.default_rng(2024)
    f = make_frame(3000, 11, score_decimals=0)
    f["tree_score"] = f["tree_score"] - 40.0                         # negative and mixed-sign scores, ties, +0.0 only
    f["filter"] = np.where(f["tree_score"] > -5, "PASS", "LOW_SCORE")
    yield "negative_scores", f, "classify", None
    n = 800
    vals = ulp_family()
    s = _spread(rng, vals, n)
    yield "ulp_apart", _frame(s, _labels(rng, n), rng.random(n) < 0.3, rng.integers(0, 14, n), _filters(rng, s, 1.0)), "classify", None
    vals = extreme_family()
    s = _spread(rng, vals, n)
    yield "subnormal_and_huge", _frame(s, _labels(rng, n), rng.random(n) < 0.3, rng.integers(0, 14, n), _filters(rng, s, 0.0)), "classify", None
    s = np.full(300, 42.0)
    yield "single_score", _frame(s, _labels(rng, 300), rng.random(300) < 0.4, rng.integers(0, 14, 300)), "classify", None
    # groups of 19, 20 and 21 called records (plus false negatives), ties at the 20th largest score
    parts = []
    for hmer, k in ((0, 19), (1, 20), (5, 21)):  # Non-hmer INDEL, HMER indel <= 4, HMER indel (4,8)
        sc = rng.permutation(np.concatenate([np.arange(30.0, 12.0, -1), [5.0, 5.0, 1.0]])[:k])  # the 20th largest: 5.0, tied
        cls = np.where(np.arange(k) % 3 == 0, "fp", "tp").astype(object)
        sc, cls = np.concatenate([sc, [1.0, 2.0]]), np.concatenate([cls, ["fn", "fn"]])
        parts.append(_frame(sc, cls, np.ones(len(sc), bool), np.full(len(sc), hmer)))
    snp = _frame(np.arange(40, dtype=np.float64) % 7, np.where(np.arange(40) % 4 == 0, "fp", "tp"))
    yield "cutoff_19_20_21", pd.concat(parts + [snp], ignore_index=True), "classify", None
    # a selection of only true calls and one of only false calls (recall of ones, precision of zeros)
    s = _round(rng.normal(10, 3, 120), 1)
    cls = np.where(np.arange(120) < 60, "tp", "fp").astype(object)
    ind = np.arange(120) >= 60
    cls[(np.arange(120) % 11 == 0) & ~ind] = "fn"
    yield "all_true_and_all_false", _frame(s, cls, ind, np.where(ind, 2, 0), _filters(rng, s, 10.0)), "classify", None
    # hmer_indel_length at every group boundary, NaN and negative, on indels and non-indels
    hv = np.array([0, 1, 4, 5, 7, 8, 10, 11, 12, 13, 20, np.nan, -1, -3])
    n = 1400
    h = _spread(rng, hv, n)
    s = _round(rng.normal(20, 8, n), 0)
    yield "hmer_boundaries", _frame(s, _labels(rng, n), rng.random(n) < 0.8, h, _filters(rng, s, 18.0)), "classify", None
    # a custom group column with values outside the seven names ("INDELS" among them: the column is not the indel flag)
    n = 900
    f = _frame(_round(rng.normal(5, 2, n), 1), _labels(rng, n), rng.random(n) < 0.4, rng.integers(0, 15, n))
    names = np.array(["SNP", "HMER indel > 12", "weird", "INDELS", "H-INDELS", "Non-hmer INDEL", "", None], dtype=object)
    f["kind"] = _spread(rng, names, n)
    yield "custom_group_outside_names", f, "classify", "kind"
    # non-indel records with hmer > 0: only H-INDELS of the indel summaries sees them
    n = 500
    ind = rng.random(n) < 0.3
    h = np.where(~ind & (rng.random(n) < 0.5), rng.integers(1, 6, n), np.where(ind, rng.integers(0, 9, n), 0))
    s = _round(rng.normal(8, 3, n), 1)
    yield "hmer_on_non_indels", _frame(s, _labels(rng, n), ind, h, _filters(rng, s, 7.0)), "classify_gt", None


def make_error_cases():
    """(name, frame, classify column, group column or None): non-finite scores, where the reference raises
    sklearn's ValueError from one function or both, or from neither."""
    base = make_frame(600, 12)
    f = base.copy()
    f.loc[np.flatnonzero(f["classify"] == "tp")[5], "tree_score"] = np.inf
    yield "inf_on_a_tp_record", f, "classify", None
    f = base.copy()
    f.loc[np.flatnonzero(f["classify"] == "fp")[3], "tree_score"] = -np.inf
    f.loc[np.flatnonzero(f["indel"] & (f["hmer_indel_length"] > 12))[0], "tree_score"] = np.inf
    yield "neg_inf_on_an_fp_record", f, "classify", None
    f = base.copy()
    f.loc[f["classify"] == "fn", "tree_score"] = np.inf                # false negatives are dropped before sklearn
    f.loc[np.flatnonzero(f["classify"] == "fn")[:3], "tree_score"] = -np.inf
    yield "inf_only_on_fn_rows", f, "classify", None
    f = base.copy()
    f["kind"] = np.where(f["indel"], "Non-hmer INDEL", "SNP").astype(object)
    row = np.flatnonzero(~f["indel"] & (f["hmer_indel_length"] == 0) & (f["classify"] == "tp"))[0]
    f.loc[row, "kind"], f.loc[row, "tree_score"] = "other", np.inf      # in no group, not an indel, no hmer
    yield "inf_in_no_group", f, "classify", "kind"
    f = base.copy()
    f["kind"] = np.where(f["indel"], "Non-hmer INDEL", "SNP").astype(object)
    row = np.flatnonzero(~f["indel"] & (f["classify"] == "fp"))[0]
    f.loc[row, ["kind", "tree_score", "hmer_indel_length"]] = ["other", np.inf, 3]
    yield "inf_only_on_an_h_indels_record", f, "classify", "kind"
