"""Test-only restatement of annotate_concordance's per-record rules (ugbio_comparison/comparison_utils.py:321-380 and
ugbio_core/vcfbed/variant_annotation.py), written row by row over Python str so that str slicing itself supplies the
sequence semantics the device kernel (csrc/conc_annotate.cu) reimplements: a negative start counts from the end, a stop
past the end is clipped, an index past the end reads "".

annotate(df, genome, flow_order, interval_beds) -> (frame, annots), with `genome` a dict contig -> str.  The interval
and filter columns use the product's host code (variantcalling_b200.concordance), which has no device part.
"""
from __future__ import annotations

import numpy as np
import pandas as pd

MOTIF, GC_WINDOW = 5, 10


def _at(seq: str, i: int) -> str:
    return seq[i:i + 1].upper()


def _run_length(seq: str, start: int) -> int:
    base, end = _at(seq, start), start + 1
    while _at(seq, end) == base:
        end += 1
    return end - start


def _hmer(seq: str | None, chrom: str, pos: int, ref: str, alleles: tuple, cls: str | None):
    if cls == "ins":
        others = [a for a in alleles if a != ref]
        if not others:
            raise IndexError("insertion without a non-REF allele")
        inserted = others[0][1:]
        if len(set(inserted)) == 1:
            if seq is None:
                raise KeyError(chrom)
            if _at(seq, pos) == inserted[0]:
                return _run_length(seq, pos), inserted[0]
    elif cls == "del":
        deleted = ref[1:]
        if len(set(deleted)) == 1:
            if seq is None:
                raise KeyError(chrom)
            if _at(seq, pos + len(ref) - 1) == deleted[0]:
                return len(deleted) + _run_length(seq, pos + len(ref) - 1), deleted[0]
    return 0, None


def _motifs(seq: str, pos: int, ref: str, indel: bool, hmer: int):
    if indel and hmer > 0:
        return seq[pos - MOTIF:pos].upper(), seq[pos + hmer:pos + hmer + MOTIF].upper()
    if indel:
        return seq[pos - MOTIF:pos].upper(), seq[pos + len(ref) - 1:pos + len(ref) - 1 + MOTIF].upper()
    return seq[pos - MOTIF - 1:pos - 1].upper(), seq[pos:pos + MOTIF].upper()


def flow_key(seq: str, flow_order: str) -> list | None:
    """Flow-space key of seq (None when a base other than ACGT is present after upper-casing)."""
    seq = seq.upper()
    if any(c not in "ACGT" for c in seq):
        return None
    key, at = [], 0
    for f in range(len(flow_order) * len(seq)):
        base = flow_order[f % len(flow_order)]
        end = at
        while end < len(seq) and seq[end] == base:
            end += 1
        key.append(end - at)
        at = end
        if at == len(seq):
            break
    return key


def cycle_skip(left: str, ref: str, alt: str, right: str, flow_order: str) -> str:
    kr, ka = flow_key(left + ref + right, flow_order), flow_key(left + alt + right, flow_order)
    if kr is None or ka is None:
        return "NA"
    if len(kr) != len(ka):
        return "cycle-skip"
    if any(a != b and (a == 0 or b == 0) for a, b in zip(kr, ka)):
        return "possible-cycle-skip"
    return "non-skip"


def annotate(df: pd.DataFrame, genome: dict, flow_order: str | None = "TGCA", interval_beds=None):
    from variantcalling_b200.concordance import _annotate_intervals, fill_filter_column

    df = df.copy()
    rows = list(zip(df["chrom"], df["pos"], df["ref"], df["alleles"], df["indel"]))
    # the passes run one after the other over all rows, so an error of an earlier pass wins over a lower row's later one
    for _chrom, _pos, ref, alleles, indel in rows:
        if indel and len(alleles) == 0:
            raise ValueError("no alleles")
    for _chrom, _pos, ref, alleles, _indel in rows:
        if len(alleles) == 0:
            raise ValueError("no alleles")
    cls = [None if not indel else ("ins" if len(ref) < max(len(a) for a in alleles) else "del")
           for _c, _p, ref, alleles, indel in rows]
    ilen = [max(abs(len(a) - len(ref)) for a in alleles) for _c, _p, ref, alleles, _i in rows]
    hm = [_hmer(genome.get(chrom), chrom, int(pos), ref, alleles, c) if indel else (0, None)
          for (chrom, pos, ref, alleles, indel), c in zip(rows, cls)]
    motifs = []
    for (chrom, pos, ref, _a, indel), (h, _n) in zip(rows, hm):
        if chrom not in genome:
            raise KeyError(chrom)
        motifs.append(_motifs(genome[chrom], int(pos), ref, bool(indel), h))
    gc = []
    for chrom, pos, _r, _a, _i in rows:
        beg = int(pos) - GC_WINDOW // 2
        window = genome[chrom][beg:beg + GC_WINDOW].upper()
        if not window:
            raise ZeroDivisionError("empty GC window")
        gc.append(float(sum(c not in "AT" for c in window)) / len(window))
    obj = lambda v: pd.Series(v, index=df.index, dtype=object)  # noqa: E731
    df["indel_classify"] = obj(cls)
    df["indel_length"] = np.array(ilen, dtype=np.int64)
    df["hmer_indel_length"] = np.array([h for h, _ in hm], dtype=np.int64)
    df["hmer_indel_nuc"] = obj([n for _, n in hm])
    df["left_motif"] = obj([m[0] for m in motifs])
    df["right_motif"] = obj([m[1] for m in motifs])
    df["gc_content"] = np.array(gc, dtype=np.float64)
    annots = []
    for bed in interval_beds or []:
        df, name = _annotate_intervals(df, bed)
        annots.append(name)
    df = fill_filter_column(df)
    if flow_order is not None:
        status = []
        for (_c, _p, ref, alleles, indel), (left, right) in zip(rows, motifs):
            if indel or len(alleles) != 2:  # noqa: PLR2004
                status.append("NA")
            else:
                status.append(cycle_skip(left, ref, alleles[1], right, flow_order))
        df["cycleskip_status"] = obj(status)
    return df, annots
