#!/usr/bin/env python
"""Generate tests/golden/concordance_annotate.json.gz from the REFERENCE's own annotate_concordance
(ugbio_comparison/comparison_utils.py:321-380 and ugbio_core/vcfbed/variant_annotation.py), run in the build
container; the fixture travels, the reference does not.

pysam, pyBigWig and simppl are not installed and none of the code exercised needs their engines, so they are
replaced by empty modules.  pyfaidx is replaced by a str-backed FASTA: fasta[contig] is a record whose [i] and [a:b]
give objects with .seq, where [i] is s[i:i + 1] (so an index past the end gives "") and [a:b] is the str slice.

Harness note: the reference is pinned to pandas < 3.  Two behaviours of that pandas are restored here: strings are
stored in object columns (future.infer_string off), and `.loc` storing a string into a float column (fill_filter_column
on a frame without a filter column) upcasts the column to object instead of raising.

Outputs: the FASTA, the BED file, the input frames, and for every case of tests/annotate_data.CASES the reference's
output frame cell by cell (column order and dtypes too); the exception type and failing row of the raising cases; the
cycle-skip table of the reference's unit test (test_variant_annotation.py:102-127) as data; and the reference's
calc_accuracy_metrics / calc_recall_precision_curve of one annotated frame with scores and classes added.
"""
import gzip
import json
import os
import sys
import types
import warnings

import numpy as np
import pandas as pd

warnings.filterwarnings("ignore")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = "/root/reference/ugbio_utils/src"
sys.path.insert(0, os.path.join(REF, "core"))
sys.path.insert(0, os.path.join(REF, "comparison"))
pd.options.future.infer_string = False

_loc_setitem = pd.core.indexing._LocIndexer.__setitem__  # noqa: SLF001


def _loc_setitem_upcasting(self, key, value):
    try:
        return _loc_setitem(self, key, value)
    except TypeError:
        obj = self.obj
        if isinstance(obj, pd.DataFrame) and isinstance(key, tuple) and len(key) == 2 and key[1] in obj.columns:  # noqa: PLR2004
            obj[key[1]] = obj[key[1]].astype(object)
            return _loc_setitem(self, key, value)
        raise


pd.core.indexing._LocIndexer.__setitem__ = _loc_setitem_upcasting  # noqa: SLF001

from tests import annotate_data as A  # noqa: E402


class _Piece:
    def __init__(self, s):
        self.seq = s


class _Record:
    def __init__(self, s):
        self.s = s

    def __len__(self):
        return len(self.s)

    def __getitem__(self, k):
        if isinstance(k, slice):
            return _Piece(self.s[k])
        return _Piece(self.s[k:k + 1])


class _Fasta(dict):
    def __init__(self, path, **k):
        super().__init__()
        name, parts = None, {}
        for ln in open(path):
            ln = ln.strip()
            if ln.startswith(">"):
                name = ln[1:].split()[0]
                parts[name] = []
            elif name:
                parts[name].append(ln)
        for k2, v in parts.items():
            self[k2] = _Record("".join(v))


class _Anything(types.ModuleType):
    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        return type(k, (), {})


class _Pyfaidx(_Anything):
    Fasta = _Fasta


sys.modules["pyfaidx"] = _Pyfaidx("pyfaidx")
for name in ("pysam", "pyBigWig", "simppl", "simppl.simple_pipeline"):
    sys.modules[name] = _Anything(name)

from ugbio_comparison import comparison_utils as ref_cmp  # noqa: E402
from ugbio_core.concordance import concordance_utils as ref_cu  # noqa: E402
from ugbio_core.vcfbed import variant_annotation as ref_va  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "concordance_annotate.json.gz")
TMP = "/tmp/golden_annotate"


def py(v):
    if isinstance(v, (tuple, list, np.ndarray)):
        return [py(x) for x in v]
    if v is None:
        return None
    if isinstance(v, (bool, np.bool_)):
        return bool(v)
    if isinstance(v, (int, np.integer)):
        return int(v)
    if isinstance(v, (float, np.floating)):
        return "NaN" if np.isnan(v) else float(v)
    return str(v)


def frame_json(df):
    return {"columns": list(df.columns), "dtypes": [str(t) for t in df.dtypes],
            "rows": [[py(v) for v in row] for row in df.itertuples(index=False, name=None)]}


def raising(df, fa, **kw):
    try:
        ref_cmp.annotate_concordance(df, fa, **kw)
    except Exception as e:  # noqa: BLE001
        return type(e).__name__
    return None


def main():
    os.makedirs(TMP, exist_ok=True)
    genome = A.make_genome()
    fa, bed = os.path.join(TMP, "ref.fa"), os.path.join(TMP, "overlaps.bed")
    open(fa, "w").write(A.fasta_text(genome))
    open(bed, "w").write(A.bed_text(genome))
    out = {"fasta": A.fasta_text(genome), "bed": A.bed_text(genome), "cases": {}, "raising": {}}
    for name, flow, with_bed, with_filter in A.CASES:
        df = A.make_frame(genome, 3000, 17, with_filter=with_filter)
        inp = frame_json(df)
        res, annots = ref_cmp.annotate_concordance(df.copy(), fa, annotate_intervals=[bed] if with_bed else None,
                                                   flow_order=flow)
        out["cases"][name] = {"flow_order": flow, "bed": with_bed, "input": inp, "output": frame_json(res),
                              "annots": annots}
        print(name, res.shape, list(res.columns)[-10:], res["cycleskip_status"].value_counts().to_dict()
              if "cycleskip_status" in res else "")

    # raising cases: one bad record inserted at a known row of a clean frame
    base = A.make_frame(genome, 40, 23)
    bad = {
        "gc_window_before_start": ("chr1", 3, "A", ("A", "C"), False),
        "gc_window_past_end": ("chrM", len(genome["chrM"]) + 6, "A", ("A", "C"), False),
        "missing_contig": ("chrZ", 100, "A", ("A", "C"), False),
        "missing_contig_hmer": ("chrZ", 100, "A", ("A", "AAA"), True),
        "no_alleles": ("chr1", 100, "A", (), False),
    }
    for name, rec in bad.items():
        for row in (7, 31):
            df = base.copy()
            df.loc[row, ["chrom", "pos", "ref", "alleles", "indel"]] = pd.Series(
                dict(zip(["chrom", "pos", "ref", "alleles", "indel"], rec)), dtype=object)
            df["pos"] = df["pos"].astype(np.int64)
            df["indel"] = df["indel"].astype(bool)
            exc = raising(df.copy(), fa)
            # the failing row: the lowest row whose removal lets the reference pass
            fail_row = None
            if exc is not None:
                for r in range(len(df)):
                    if raising(df.drop(index=r).reset_index(drop=True), fa) is None:
                        fail_row = r
                        break
            out["raising"][f"{name}@{row}"] = {"input": frame_json(df), "exception": exc, "row": fail_row}
            print("raising", name, row, exc, fail_row)

    # cycle-skip table of test_variant_annotation.py:102-127
    table = []
    for left, ref, alt, right, flow in [
        ("CA", "T", "C", "AT", "TGCA"), ("CA", "T", "G", "AT", "TGCA"), ("CA", "T", "A", "AT", "TGCA"),
        ("GT", "A", "C", "GA", "TGCA"), ("GT", "A", "G", "GA", "TGCA"), ("TT", "G", "A", "CC", "TGCA"),
        ("AC", "G", "T", "TG", "TACG"), ("AC", "G", "N", "TG", "TGCA"), ("AAAAA", "C", "G", "TTTTT", "TGCA"),
        ("CCCCC", "A", "T", "GGGGG", "TGC"),
    ]:
        df = pd.DataFrame({"indel": [False], "alleles": [(ref, alt)], "left_motif": [left], "ref": [ref],
                           "right_motif": [right]})
        table.append({"left": left, "ref": ref, "alt": alt, "right": right, "flow_order": flow,
                      "status": ref_va.annotate_cycle_skip(df, flow)["cycleskip_status"][0]})
    out["cycle_skip_table"] = table

    # metrics of one annotated frame
    df = A.make_frame(genome, 3000, 29)
    res, _ = ref_cmp.annotate_concordance(df.copy(), fa)
    rng = np.random.default_rng(29)
    scores = np.round(rng.random(len(res)), 3)
    classes = np.array(["tp", "fp", "fn"], dtype=object)[rng.integers(0, 3, len(res))]
    # every variant group gets a true call, so that each curve has a positive class
    groups = res["indel"].astype(int) * (1 + np.minimum(res["hmer_indel_length"].to_numpy(), 13))
    for g in np.unique(groups):
        classes[np.flatnonzero(groups == g)[0]] = "tp"
    met = res.copy()
    met["tree_score"] = scores
    met["classify"] = classes
    acc = ref_cu.calc_accuracy_metrics(met.copy(), "classify")
    curve = ref_cu.calc_recall_precision_curve(met.copy(), "classify")
    out["metrics"] = {"input": frame_json(df), "tree_score": scores.tolist(), "classify": classes.tolist(),
                      "accuracy": {c: py(list(acc[c])) for c in acc.columns},
                      "curve": {c: py(list(curve[c])) for c in curve.columns}}
    with gzip.open(OUT, "wt", compresslevel=9) as fh:
        json.dump(out, fh)
    print("wrote", OUT, os.path.getsize(OUT) >> 10, "KiB")


if __name__ == "__main__":
    main()
