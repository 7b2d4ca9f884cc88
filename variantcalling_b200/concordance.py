"""Precision / recall of a filtered call set against truth (BASELINE.json configs[4]) -- host
mirror of ``ugbio_core/concordance/concordance_utils.py``: same function names, arguments, output
frames and error behaviour; the per-record work (group selection, tp/fp/fn counts, the sort +
cumulative counts behind the precision-recall curves) runs in ``csrc/concordance.cu`` through the
C ABI (``ugvc_conc_*``).  There is no CPU path: without a CUDA device ``ConcordanceContext``
raises.

  calc_accuracy_metrics(df, classify_column_name, ignored_filters=None, group_testing_column_name=None)
      -> concordance_utils.py:11-106
  calc_recall_precision_curve(...)                 -> :109-188
  get_concordance_metrics(predictions, scores, truth, fn_mask, ...)   -> :346-458
  annotate_concordance(concordance_df, fasta, ...)  -> ugbio_comparison/comparison_utils.py:321-380 (the per-record
      passes in ``csrc/conc_annotate.cu``; interval and filter columns in NumPy / pandas)
"""
from __future__ import annotations

import ctypes as C
import itertools
import logging
import os
from collections import OrderedDict

import numpy as np
import pandas as pd

from variantcalling_b200 import lib
from variantcalling_b200.multiallelics import read_fasta_contig

logger = logging.getLogger(__name__)

# ugvc_conc_run writes N_GROUPS x N_COUNTERS: the six metric counters (tp, fp, missed, initial_tp, n_called, n_fn),
# then the NaN and +-inf scores among the called records
N_GROUPS, N_COUNTERS, N_METRIC_COUNTERS = 9, 8, 6
CLASS_CODE = {"fp": 0, "tp": 1, "fn": 2, "tn": 3}
METRIC_COLUMNS = ["tp", "fp", "fn", "precision", "recall", "f1", "initial_tp", "initial_fp", "initial_fn",
                  "initial_precision", "initial_recall", "initial_f1"]


def get_selection_functions() -> OrderedDict:
    """concordance_utils.py:266-275 (the GPU derives the same groups from indel / hmer_indel_length)."""
    sfs = OrderedDict()
    sfs["SNP"] = lambda x: np.logical_not(x.indel)
    sfs["Non-hmer INDEL"] = lambda x: x.indel & (x.hmer_indel_length == 0)
    sfs["HMER indel <= 4"] = lambda x: x.indel & (x.hmer_indel_length > 0) & (x.hmer_indel_length < 5)  # noqa: PLR2004
    sfs["HMER indel (4,8)"] = lambda x: x.indel & (x.hmer_indel_length >= 5) & (x.hmer_indel_length < 8)  # noqa: PLR2004
    sfs["HMER indel [8,10]"] = lambda x: x.indel & (x.hmer_indel_length >= 8) & (x.hmer_indel_length <= 10)  # noqa: PLR2004
    sfs["HMER indel 11,12"] = lambda x: x.indel & (x.hmer_indel_length >= 11) & (x.hmer_indel_length <= 12)  # noqa: PLR2004
    sfs["HMER indel > 12"] = lambda x: x.indel & (x.hmer_indel_length > 12)  # noqa: PLR2004
    return sfs


GROUP_NAMES = list(get_selection_functions().keys())


def init_metrics_df() -> pd.DataFrame:
    return pd.DataFrame(columns=["group"] + METRIC_COLUMNS)


def convert_filter2call(filter_str: str, ignored_filters: set | None = None) -> str:
    """concordance_utils.py:228-243 -- the reference resets ``ignored_filters`` to {"PASS"} (:242),
    so only PASS counts as a call whatever the caller passes; kept."""
    ignored_filters = {"PASS"}
    return "tp" if all(_filter in ignored_filters for _filter in filter_str.split(";")) else "fp"


def get_precision(false_positives, true_positives, return_if_denominator_is_0=1):
    if false_positives + true_positives == 0:
        return return_if_denominator_is_0
    return 1 - false_positives / (false_positives + true_positives)


def get_recall(false_negatives, true_positives, return_if_denominator_is_0=1):
    if false_negatives + true_positives == 0:
        return return_if_denominator_is_0
    return 1 - false_negatives / (false_negatives + true_positives)


def get_f1(precision, recall, null_value=np.nan):
    if null_value in {precision, recall}:
        return null_value
    return 0 if precision + recall == 0 else 2 * precision * recall / (precision + recall)


class ConcordanceContext:
    """Owns a ``ugvc_conc`` handle (one per GPU)."""

    def __init__(self, device: int = 0):
        self.lib = lib.load_library()
        h = C.c_void_p()
        rc = self.lib.ugvc_conc_create(device, C.byref(h))
        if rc != 0:
            raise lib.UgvcError(rc, self.lib.ugvc_conc_last_error(None).decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.ugvc_conc_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001, S110
            pass

    def launch_count(self) -> int:
        return int(self.lib.ugvc_conc_launch_count(self.h))

    def run(self, scores, pred, cls, indel, hmer, group=None, want_curves=True) -> dict:
        """Arrays of one length -> dict(counts (9, 6), non_finite (9, 2): NaN / inf scores of called records,
        curve_len, cutoff, selected (9, 2))."""
        n = len(scores)
        scores = np.ascontiguousarray(scores, dtype=np.float64)
        pred = np.ascontiguousarray(pred, dtype=np.uint8)
        cls = np.ascontiguousarray(cls, dtype=np.uint8)
        indel = np.ascontiguousarray(indel, dtype=np.uint8)
        hmer = np.ascontiguousarray(hmer, dtype=np.int32)
        group = None if group is None else np.ascontiguousarray(group, dtype=np.int8)
        for a in (pred, cls, indel, hmer) + (() if group is None else (group,)):
            if len(a) != n:
                raise ValueError("concordance columns differ in length")
        counts = np.zeros((N_GROUPS, N_COUNTERS), dtype=np.int64)
        curve_len = np.zeros(N_GROUPS, dtype=np.int64)
        cutoff = np.zeros(N_GROUPS, dtype=np.float64)
        selected = np.zeros((N_GROUPS, 2), dtype=np.int64)
        p = lib._ptr  # noqa: SLF001
        rc = self.lib.ugvc_conc_run(self.h, n, p(scores), p(pred), p(cls), p(indel), p(hmer), p(group), 0,
                                    int(want_curves), p(counts), p(curve_len), p(cutoff), p(selected))
        if rc != 0:
            raise lib.UgvcError(rc, self.lib.ugvc_conc_last_error(self.h).decode())
        return {"counts": counts[:, :N_METRIC_COUNTERS].copy(), "non_finite": counts[:, N_METRIC_COUNTERS:].copy(),
                "curve_len": curve_len, "cutoff": cutoff, "selected": selected}

    def classify(self, gt_ultima, gt_truth, base=None) -> tuple[np.ndarray, np.ndarray]:
        """The `classify` / `classify_gt` columns of vcf2concordance (comparison_utils.py:153-229) for genotype tuples
        (None alleles allowed, one or two alleles) and vcfeval's BASE column; string arrays "tp" / "fp" / "fn"."""
        n = len(gt_ultima)

        def pack(gts):
            out = np.full((n, 2), -2, dtype=np.int8)
            for i, g in enumerate(gts):
                g = tuple(g)
                if len(g) > 2:  # noqa: PLR2004
                    raise ValueError("genotypes of more than two alleles are not lowered")
                for k, a in enumerate(g):
                    out[i, k] = -1 if a is None else int(a)
            return np.ascontiguousarray(out)

        gu, gt = pack(gt_ultima), pack(gt_truth)
        bfn = None if base is None else np.ascontiguousarray(np.isin(np.asarray(base, dtype=object), ["FN", "FN_CA"]).astype(np.uint8))
        c, g = np.empty(n, dtype=np.uint8), np.empty(n, dtype=np.uint8)
        rc = self.lib.ugvc_conc_classify(self.h, n, lib._ptr(gu), lib._ptr(gt), lib._ptr(bfn), lib._ptr(c), lib._ptr(g))  # noqa: SLF001
        if rc:
            raise lib.UgvcError(rc, self.lib.ugvc_conc_last_error(self.h).decode())
        names = np.array(["tp", "fp", "fn"], dtype=object)
        return names[c], names[g]

    def curve(self, g: int, n: int):
        """Raw curve of group g: (precision, recall, thresholds), increasing thresholds."""
        out = [np.empty(max(1, n), dtype=np.float64) for _ in range(3)]
        rc = self.lib.ugvc_conc_curve(self.h, g, lib._ptr(out[0]), lib._ptr(out[1]), lib._ptr(out[2]), out[0].size)  # noqa: SLF001
        if rc != 0:
            raise lib.UgvcError(rc, self.lib.ugvc_conc_last_error(self.h).decode())
        return tuple(a[:n] for a in out)


    def annot_contig(self, fasta: str, contig: str) -> int:
        """Id of `contig` of `fasta` on the handle (-1 when the FASTA lacks it), read and uploaded on first use."""
        lib.load_annotation()
        key = (os.path.abspath(fasta), contig)
        cache = self.__dict__.setdefault("_annot_contigs", {})
        if key not in cache:
            try:
                seq = read_fasta_contig(fasta, contig, as_bytes=True)
            except KeyError:
                cache[key] = -1
                return -1
            buf = np.frombuffer(seq, dtype=np.uint8) if seq else np.zeros(1, np.uint8)
            cid = C.c_int32()
            rc = self.lib.ugvc_conc_annot_add_contig(self.h, lib._ptr(buf), len(seq), C.byref(cid))  # noqa: SLF001
            if rc != 0:
                raise lib.UgvcError(rc, self.lib.ugvc_conc_last_error(self.h).decode())
            cache[key] = int(cid.value)
        return cache[key]

    def annotate(self, contig_ids, pos, indel, refs, alleles, flow_order: str | None, motif_size: int = 5,
                 gc_window: int = 10) -> dict:
        """The per-record columns of annotate_concordance as typed arrays (see ugvc_conc_annotate).  refs: sequence of
        str, alleles: sequence of tuples of str, ASCII.  Raises what the reference raises, at the same record."""
        lib.load_annotation()
        n = len(refs)
        contig_ids = np.ascontiguousarray(contig_ids, dtype=np.int32)
        pos = np.ascontiguousarray(pos, dtype=np.int64)
        indel = np.ascontiguousarray(indel, dtype=np.uint8)
        n_alleles = np.fromiter(map(len, alleles), dtype=np.int64, count=n)
        empty = np.flatnonzero(n_alleles == 0)
        if len(empty):  # max() of no alleles: classify_indel's indel rows fail first, then indel_length's
            bad = np.flatnonzero((n_alleles == 0) & (indel != 0))
            row = int(bad[0] if len(bad) else empty[0])
            raise ValueError(f"record {row}: max() iterable argument is empty (a record without alleles)")
        ref_bytes, ref_off = _pack_strings(refs)
        flat = list(itertools.chain.from_iterable(alleles))
        al_bytes, al_off = _pack_strings(flat)
        rec_off = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(n_alleles, out=rec_off[1:])
        out = {"class": np.empty(n, np.int8), "indel_length": np.empty(n, np.int32), "hmer_length": np.empty(n, np.int32),
               "hmer_nuc": np.empty(n, np.uint8), "left": np.zeros((n, motif_size), np.uint8),
               "right": np.zeros((n, motif_size), np.uint8), "left_len": np.empty(n, np.uint8),
               "right_len": np.empty(n, np.uint8), "gc": np.empty(n, np.float64),
               "cycleskip": np.empty(n, np.int8) if flow_order is not None else None}
        p = lib._ptr  # noqa: SLF001
        fo = None if flow_order is None else flow_order.encode("ascii")
        rc = self.lib.ugvc_conc_annotate(self.h, n, p(contig_ids), p(pos), p(indel), p(ref_bytes), p(ref_off),
                                         p(al_bytes), p(al_off), p(rec_off), fo, motif_size, gc_window, p(out["class"]),
                                         p(out["indel_length"]), p(out["hmer_length"]), p(out["hmer_nuc"]), p(out["left"]),
                                         p(out["right"]), p(out["left_len"]), p(out["right_len"]), p(out["gc"]),
                                         p(out["cycleskip"]))
        if rc == lib.UGVC_E_DATA:
            row, reason = C.c_int64(), C.c_int()
            self.lib.ugvc_conc_annot_error(self.h, C.byref(row), C.byref(reason))
            raise AnnotationDataError(int(row.value), int(reason.value))
        if rc != 0:
            raise lib.UgvcError(rc, self.lib.ugvc_conc_last_error(self.h).decode())
        return out


class AnnotationDataError(Exception):
    """A record where the reference's annotate_concordance raises: `row` and the UGVC_ANNOT_E_* `reason`."""

    def __init__(self, row: int, reason: int):
        super().__init__(row, reason)
        self.row, self.reason = row, reason


def _pack_strings(strs) -> tuple[np.ndarray, np.ndarray]:
    """Sequence of ASCII str -> (bytes as uint8, int64 offsets of len + 1)."""
    lens = np.fromiter(map(len, strs), dtype=np.int64, count=len(strs))
    data = "".join(strs).encode("ascii")
    off = np.zeros(len(strs) + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    return (np.frombuffer(data, dtype=np.uint8) if data else np.zeros(1, np.uint8)), off


_default_ctx: ConcordanceContext | None = None


def _context(ctx: ConcordanceContext | None) -> ConcordanceContext:
    global _default_ctx  # noqa: PLW0603
    if ctx is not None:
        return ctx
    if _default_ctx is None:
        _default_ctx = ConcordanceContext(0)
    return _default_ctx


def _metrics_from_counts(c: np.ndarray) -> dict:
    """get_concordance_metrics' scalar part (:418-447) from the six device counters of a group."""
    tp, fp, missed, itp, n_called, n_fn = (int(v) for v in c)
    if n_called == 0:  # len(predictions) == 0 after dropping the false negatives -> the "empty" row (:323-338)
        m = dict.fromkeys(METRIC_COLUMNS, 1.0)
        for k in ("tp", "fp", "fn", "initial_tp", "initial_fp", "initial_fn"):
            m[k] = 0
        return m
    fn = n_fn + missed
    ifp = n_called - itp
    precision, recall = get_precision(fp, tp), get_recall(fn, tp)
    iprecision, irecall = get_precision(ifp, itp), get_recall(n_fn, itp)
    return {"tp": tp, "fp": fp, "fn": fn, "precision": precision, "recall": recall, "f1": get_f1(precision, recall),
            "initial_tp": itp, "initial_fp": ifp, "initial_fn": n_fn, "initial_precision": iprecision,
            "initial_recall": irecall, "initial_f1": get_f1(iprecision, irecall)}


def _raise_on_non_finite(called_scores: np.ndarray, res: dict, groups, dtype) -> None:
    """sklearn's assert_all_finite on the called scores of each group the reference draws a curve for (it draws one
    even when only the metrics are returned), in its order: the first group with a NaN or an infinity raises, NaN's
    message before inf's.  Whether any called score is non-finite is one pass over the host column; which group
    meets it first comes from the device's per-group tallies.  dtype is the score column's, which sklearn names."""
    if np.isfinite(called_scores).all():
        return
    for g in groups:
        n_nan, n_inf = (int(v) for v in res["non_finite"][g])
        if n_nan:
            raise ValueError("Input contains NaN.")
        if n_inf:
            raise ValueError(f"Input contains infinity or a value too large for {dtype!r}.")


def _score_dtype(scores) -> np.dtype:
    dt = getattr(scores, "dtype", None)
    return dt if dt is not None and dt.kind == "f" else np.dtype(np.float64)


def _curve_from_device(ctx: ConcordanceContext, g: int, res: dict) -> dict:
    """stats_utils.precision_recall_curve :141-210 after the sklearn call, and the threshold choice of
    get_concordance_metrics :391-407, from the raw device curve of group g."""
    n_called, n_fn = int(res["counts"][g, 4]), int(res["counts"][g, 5])
    empty = np.array([])
    if n_called + n_fn == 0:
        return {"predictions": empty, "precision": empty, "recall": empty, "f1": empty, "threshold": 0}
    if n_called == 0:
        # only false negatives: the reference goes on with [nan, 1] / [1, 0] / [0], which the [1:-1]
        # trimming empties, and get_concordance_metrics then returns its "empty curve" row (:409-416)
        return {"threshold": 0, "predictions": [], "precision": [], "recall": [], "f1": []}
    raw_p, raw_r, thr = ctx.curve(g, int(res["curve_len"][g]))
    sel_true = int(res["selected"][g, 1])
    with np.errstate(invalid="ignore"):  # no true call and no false negative: NaN recalls, as NumPy gives the reference
        correction = np.float64(sel_true) / np.float64(sel_true + n_fn)
    # sklearn appends (1, 0) to precision / recall; the reference then drops the first and last points
    recalls = (np.hstack((raw_r, 0)) * correction)[1:-1]
    precisions = np.hstack((raw_p, 1))[1:-1]
    thr = thr[1:]
    f1 = 2 * (recalls * precisions) / (recalls + precisions + np.finfo(float).eps)
    keep = ~(thr > res["cutoff"][g])
    precisions, recalls, f1, thr = precisions[keep], recalls[keep], f1[keep], thr[keep]
    threshold = thr[np.argmax(f1)] if len(f1) > 0 else 0
    return {"predictions": thr, "precision": precisions, "recall": recalls, "f1": f1, "threshold": threshold}


def get_concordance_metrics(predictions, scores, truth, fn_mask, *, return_metrics=True, return_curves=True,
                            ctx: ConcordanceContext | None = None):
    """concordance_utils.py:346-458 on one selection (everything lands in group 0 on the device)."""
    assert return_curves or return_metrics, "At least one of return_curves or return_metrics should be True"  # noqa: S101
    ctx = _context(ctx)
    truth = np.asarray(truth)
    fn_mask = np.asarray(fn_mask, dtype=bool)
    cls = np.where(fn_mask, 2, np.where(truth > 0, 1, 0)).astype(np.uint8)
    n = len(cls)
    res = ctx.run(scores, np.asarray(predictions) > 0, cls, np.zeros(n, np.uint8), np.zeros(n, np.int32),
                  group=np.zeros(n, np.int8), want_curves=return_curves)
    scores = np.asarray(scores)
    _raise_on_non_finite(np.asarray(scores[~fn_mask], dtype=np.float64), res, [0], _score_dtype(scores))
    metrics_df = pd.DataFrame(_metrics_from_counts(res["counts"][0]), index=[0])
    if not return_curves:
        return metrics_df
    curve_df = pd.DataFrame(pd.Series(_curve_from_device(ctx, 0, res))).T
    return (metrics_df, curve_df) if return_metrics else curve_df


def validate_preprocess_concordance(concordance_df: pd.DataFrame, group_testing_column_name: str | None = None):
    """concordance_utils.py:191-225"""
    assert "tree_score" in concordance_df.columns, "Input concordance file should be after applying a model"  # noqa: S101
    concordance_df.loc[pd.isna(concordance_df["hmer_indel_nuc"]), "hmer_indel_nuc"] = "N"
    if np.any(pd.isna(concordance_df["filter"])):
        logger.warning("Null values in filter column (n=%i). Setting them as PASS, but it is suspicious",
                       pd.isna(concordance_df["filter"]).sum())
        concordance_df.loc[pd.isna(concordance_df["filter"]), "filter"] = "PASS"
    if np.any(pd.isna(concordance_df["tree_score"])):
        logger.warning("Null values in concordance dataframe tree_score (n=%i). Setting them as zero, but it is suspicious",
                       pd.isna(concordance_df["tree_score"]).sum())
        concordance_df.loc[pd.isna(concordance_df["tree_score"]), "tree_score"] = 0
    if group_testing_column_name is not None:
        concordance_df["group_testing"] = concordance_df[group_testing_column_name]
        removed = pd.isna(concordance_df["group_testing"])
        logger.info("Removing %i/%i variants with no type", removed.sum(), concordance_df.shape[0])
        concordance_df = concordance_df[~removed]
    return concordance_df


def _device_pass(concordance_df, classify_column_name, group_testing_column_name, ctx, *, want_curves):
    df = validate_preprocess_concordance(concordance_df, group_testing_column_name)
    filters = df["filter"]
    calls = {f: convert_filter2call(f) == "tp" for f in pd.unique(filters)}
    pred = filters.map(calls).to_numpy(dtype=bool)
    labels = df[classify_column_name]
    unknown = set(pd.unique(labels)) - set(CLASS_CODE)
    if unknown:
        raise ValueError(f"unexpected values in {classify_column_name}: {sorted(map(str, unknown))}")
    cls = labels.map(CLASS_CODE).to_numpy(dtype=np.uint8)
    hmer = df["hmer_indel_length"].to_numpy(dtype=np.float64)
    hmer = np.where(np.isnan(hmer), -1, hmer).astype(np.int32)
    group = None
    if group_testing_column_name is not None:
        ids = {name: i for i, name in enumerate(GROUP_NAMES)}
        group = df["group_testing"].map(lambda v: ids.get(v, -1)).to_numpy(dtype=np.int8)
    ctx = _context(ctx)
    scores = df["tree_score"].to_numpy(dtype=np.float64)
    res = ctx.run(scores, pred, cls, df["indel"].to_numpy(dtype=bool), hmer, group=group, want_curves=want_curves)
    # calc_accuracy_metrics draws the curves of the 7 groups, INDELS and H-INDELS; calc_recall_precision_curve of
    # all but H-INDELS
    _raise_on_non_finite(scores[cls != CLASS_CODE["fn"]], res, range(N_GROUPS - 1) if want_curves else range(N_GROUPS),
                         _score_dtype(df["tree_score"]))
    return ctx, res


def calc_accuracy_metrics(concordance_df: pd.DataFrame, classify_column_name: str, ignored_filters=None,
                          group_testing_column_name: str | None = None, ctx: ConcordanceContext | None = None):
    """concordance_utils.py:11-106: one row per variant group, then INDELS and H-INDELS, rounded to 5 decimals."""
    _ctx, res = _device_pass(concordance_df, classify_column_name, group_testing_column_name, ctx, want_curves=False)
    rows = []
    for g, name in enumerate(GROUP_NAMES + ["INDELS", "H-INDELS"]):
        rows.append({"group": name, **_metrics_from_counts(res["counts"][g])})
    return pd.DataFrame(rows, columns=["group"] + METRIC_COLUMNS).round(5)


def calc_recall_precision_curve(concordance_df: pd.DataFrame, classify_column_name: str, ignored_filters=None,
                                group_testing_column_name: str | None = None, ctx: ConcordanceContext | None = None):
    """concordance_utils.py:109-188: curves of the variant groups and of INDELS."""
    ctx, res = _device_pass(concordance_df, classify_column_name, group_testing_column_name, ctx, want_curves=True)
    rows = []
    for g, name in enumerate(GROUP_NAMES + ["INDELS"]):
        c = _curve_from_device(ctx, g, res)
        rows.append({"group": name, "precision": c["precision"], "recall": c["recall"], "f1": c["f1"],
                     "threshold": c["threshold"], "predictions": c["predictions"]})
    return pd.DataFrame(rows, columns=["group", "precision", "recall", "f1", "threshold", "predictions"])


# ------------------------------------------------------------------ annotate_concordance (comparison_utils.py:321-380)
ANNOT_MOTIF_SIZE, ANNOT_GC_WINDOW = 5, 10
_INDEL_CLASS = np.array([None, "ins", "del"], dtype=object)
_CYCLE_SKIP = np.array(["NA", "cycle-skip", "possible-cycle-skip", "non-skip"], dtype=object)
_HMER_NUC = np.array([None] + [chr(b) for b in range(1, 256)], dtype=object)


def _object_column(values: np.ndarray, index) -> pd.Series:
    return pd.Series(values, index=index, dtype=object)


def _motif_strings(buf: np.ndarray) -> np.ndarray:
    """(n, size) zero-padded upper-case motif bytes -> object array of str."""
    if buf.shape[1] == 0:
        return np.full(buf.shape[0], "", dtype=object)
    return np.ascontiguousarray(buf).view(f"S{buf.shape[1]}").ravel().astype(f"U{buf.shape[1]}").astype(object)


def _raise_like_the_reference(err: AnnotationDataError, chrom: np.ndarray):
    """The exception the reference raises at err.row (chained to err, which carries the row)."""
    row = err.row
    if err.reason == 1:
        raise IndexError(f"record {row}: list index out of range (an insertion whose alleles all equal ref)") from err
    if err.reason == 2:  # noqa: PLR2004
        raise KeyError(chrom[row]) from err
    if err.reason == 3:  # noqa: PLR2004
        raise ZeroDivisionError(f"record {row}: float division by zero (empty GC window)") from err
    raise RuntimeError(f"record {row}: annotation error {err.reason}") from err


def fill_filter_column(df: pd.DataFrame) -> pd.DataFrame:
    """variant_annotation.py:593-612: missing and empty FILTER values become PASS.  A column created here (or one of
    NaN only) turns into an object column, as the reference's pandas does when it stores a string in a float column."""
    if "filter" not in df.columns:
        df["filter"] = np.nan
    fill = pd.isna(df["filter"]) | (df["filter"] == "")
    if fill.any() and df["filter"].dtype.kind == "f":
        df["filter"] = df["filter"].astype(object)
    df.loc[fill, "filter"] = "PASS"
    return df


def _annotate_intervals(df: pd.DataFrame, annotfile: str) -> tuple[pd.DataFrame, str]:
    """variant_annotation.py:549-590: a boolean column named after the BED file, True where a record's pos falls in an
    interval.  The intervals are sorted by (chromosome, start) only and both NumPy searches run on that order, as in
    the reference, so overlapping intervals give the reference's answer rather than an exact containment test."""
    annot = annotfile.split("/")[-1]
    if annot.endswith(".bed"):
        annot = annot[:-4]
    df[annot] = False
    bed = pd.read_csv(annotfile, names=["chromosome", "start", "end"], usecols=[0, 1, 2], index_col=None, sep="\t")
    bed = bed.sort_values(["chromosome", "start"])
    bed["chromosome"] = bed["chromosome"].astype("string")
    bed_rows = bed.groupby("chromosome").groups
    for chrom, rows in df.groupby("chrom").groups.items():
        if chrom not in bed_rows:
            continue
        pos = np.array(df.loc[rows, "pos"])
        after_start = np.searchsorted(np.array(bed.loc[bed_rows[chrom], "start"]), pos) - 1
        before_end = np.searchsorted(np.array(bed.loc[bed_rows[chrom], "end"]), pos)
        df.loc[rows, annot] = after_start == before_end
    return df, annot


def annotate_concordance(concordance_df: pd.DataFrame, fasta: str, bw_high_quality: list[str] | None = None,
                         bw_all_quality: list[str] | None = None, annotate_intervals: list[str] | None = None,
                         flow_order: str | None = "TGCA", ctx: ConcordanceContext | None = None,
                         ) -> tuple[pd.DataFrame, list]:
    """comparison_utils.py:321-380.  Adds, in the reference's order, indel_classify, indel_length, hmer_indel_length,
    hmer_indel_nuc, left_motif, right_motif, gc_content (one kernel launch over all records), one boolean column per
    interval file, fills `filter`, and adds cycleskip_status when flow_order is not None.  The frame is changed in place
    and returned with the list of interval column names.  Coverage from bigWig files is not supported."""
    interval_files = [] if annotate_intervals is None else annotate_intervals
    if bw_all_quality is not None and bw_high_quality is not None:
        raise NotImplementedError("coverage from bigWig files (get_coverage) is not supported")
    df = concordance_df
    ctx = _context(ctx)
    codes, names = pd.factorize(df["chrom"], use_na_sentinel=False)
    ids = np.array([ctx.annot_contig(fasta, str(c)) for c in names], dtype=np.int32)
    chrom = np.asarray(names, dtype=object)[codes]
    try:
        res = ctx.annotate(ids[codes] if len(ids) else np.zeros(0, np.int32), df["pos"].to_numpy(dtype=np.int64),
                           df["indel"].to_numpy(dtype=bool), df["ref"].tolist(), df["alleles"].tolist(), flow_order,
                           ANNOT_MOTIF_SIZE, ANNOT_GC_WINDOW)
    except AnnotationDataError as e:
        _raise_like_the_reference(e, chrom)
    idx = df.index
    df["indel_classify"] = _object_column(_INDEL_CLASS[res["class"]], idx)
    df["indel_length"] = res["indel_length"].astype(np.int64)
    df["hmer_indel_length"] = res["hmer_length"].astype(np.int64)
    df["hmer_indel_nuc"] = _object_column(_HMER_NUC[res["hmer_nuc"]], idx)
    df["left_motif"] = _object_column(_motif_strings(res["left"]), idx)
    df["right_motif"] = _object_column(_motif_strings(res["right"]), idx)
    df["gc_content"] = res["gc"]
    annots = []
    for path in interval_files:
        df, annot = _annotate_intervals(df, path)
        annots.append(annot)
    df = fill_filter_column(df)
    if flow_order is not None:
        df["cycleskip_status"] = _object_column(_CYCLE_SKIP[res["cycleskip"]], idx)
    return df, annots
