"""ORACLE (test infrastructure, not product code).

gvcf_hcr (``ugvc/joint/gvcf_bed.py:gvcf_to_bed``, ``ugvc/pipelines/vcfbed/gvcf_hcr_main.py``) restated over text, for the
tests of the device path (DESIGN.md 4e):

* each record's interval: ``start = POS - 1``; ``end`` = htslib's ``record.stop`` (INFO/END when the header declares it,
  the first ``END=`` of 1..10 digits, and it lies beyond ``start``; else ``start + len(REF)``); a RefCall deletion
  (``len(REF) > 1`` and sample 0 without GQ, or GT ``(0, 0)`` / ``(None, None)``) ends at ``start + 1`` -- GT is read only
  there, ``KeyError`` when the FORMAT lacks it;
* the skip rule, in the reference's own words (``chrom == last_chrom and start < extent``);
* the selection of a kept record on sample 0's GQ with Python's short circuit, typed as ``oracle/vcf_reader.py`` types
  values (Number=1 a scalar, any other Number a tuple, undeclared or String a str, ``.`` / a dropped sub-field None /
  (None,)): ``TypeError`` where a None, a tuple or a str is compared;
* the stances: a GQ / GT literal that cannot be typed raises (``"literal"``) at its record whether or not it is read; POS
  decreasing within a contig or a contig that comes back raises ``ValueError`` (``"unsorted"``);
* ``merge``: bedtools merge's default rule (``-d 0``: an interval that starts at or before the end of the current one
  on the same chrom extends it).  Parity-unpinned: bedtools is not installed here.

``tests/golden/gvcf_hcr.json.gz`` (scripts/make_golden_gvcf_hcr.py) pins gvcf_to_bed to the reference's own function.
"""
from __future__ import annotations

import re

import numpy as np

from oracle.vcf_reader import OracleHeader

_INT = re.compile(r"[+-]?[0-9]{1,18}")
_FLOAT = re.compile(r"[+-]?([0-9]+\.?[0-9]*([eE][+-]?[0-9]+)?|\.[0-9]+([eE][+-]?[0-9]+)?|nan|inf|infinity)", re.IGNORECASE)
_END = re.compile(r"[0-9]{1,10}")
_ALLELE = re.compile(r"[0-9]{1,9}")


class LiteralError(ValueError):
    """A GQ / GT literal that cannot be typed (the product raises UgvcDataError for the record)."""


class UnsortedError(ValueError):
    """POS decreases within a contig, or a contig's records are not contiguous."""


def gq_decl(header: OracleHeader):
    """How GQ is typed: ("String", None) when undeclared or of another Type, else (Number, Type)."""
    if "GQ" not in header.formats:
        return ("String", None)
    number, vtype = header.formats["GQ"]
    if vtype not in ("Integer", "Float"):
        return ("String", None)
    return (number, vtype)


def _elem(text: str, vtype: str):
    if text == ".":
        return None
    if vtype == "Integer":
        if not _INT.fullmatch(text):
            raise LiteralError(text)
        return int(text)
    if not _FLOAT.fullmatch(text):
        raise LiteralError(text)
    return float(np.float32(float(text)))


def typed_gq(text: str | None, decl):
    number, vtype = decl
    if number == "String":
        return text
    if text is None or text == ".":
        return None if number == "1" else (None,)
    if text == "":
        return None if number == "1" else ()
    if number == "1":
        return _elem(text, vtype)
    return tuple(_elem(t, vtype) for t in text.split(","))


def typed_gt(text: str | None):
    if text is None:
        return (None,)
    out = []
    for tok in re.split(r"[/|]", text):
        if tok in ("", "."):
            out.append(None)
        elif _ALLELE.fullmatch(tok):
            out.append(int(tok))
        else:
            raise LiteralError(text)
    return tuple(out)


class Sample0:
    """sample 0 as pysam's VariantRecordSample answers ``in`` and ``[]``: a key is in it when the record's FORMAT names
    it; GQ / GT typed when the record is read."""

    def __init__(self, cols: list[str], decl):
        keys = cols[8].split(":") if len(cols) > 8 and cols[8] != "." else []  # noqa: PLR2004
        vals = cols[9].split(":") if len(cols) > 9 else None  # noqa: PLR2004
        self.values = {}
        for key in ("GQ", "GT"):
            if key in keys:
                i = keys.index(key)
                text = vals[i] if vals is not None and i < len(vals) else None
                self.values[key] = typed_gq(text, decl) if key == "GQ" else typed_gt(text)

    def __contains__(self, key):
        return key in self.values

    def __getitem__(self, key):
        if key not in self.values:
            raise KeyError(f"invalid FORMAT: {key}")
        return self.values[key]


class Record:
    """The attributes gvcf_to_bed reads: chrom, start, stop, ref, samples[0]."""

    def __init__(self, line: str, decl, info_end: bool):
        cols = line.split("\t")
        self.chrom, self.pos, self.ref = cols[0], int(cols[1]), cols[3]
        self.start = self.pos - 1
        self.stop = self.start + max(1, len(self.ref))
        if info_end and cols[7] != ".":
            for kv in cols[7].split(";"):
                if kv.startswith("END="):
                    if _END.fullmatch(kv[4:]) and int(kv[4:]) > self.start:
                        self.stop = int(kv[4:])
                    break
        self.samples = [Sample0(cols, decl)]


def records(text: str):
    """(header, data lines) of VCF text."""
    lines = text.split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    head = [ln for ln in lines if ln.startswith("#")]
    return OracleHeader(head), [ln for ln in lines if ln and not ln.startswith("#")]


def iterate(text: str):
    """The records of VCF text in file order, as pysam's fetch() yields them (typing errors raised when a record is
    read), with the unsorted stances checked."""
    header, data = records(text)
    decl, info_end = gq_decl(header), "END" in header.info
    seen, last, last_pos = set(), None, -1
    for ln in data:
        rec = Record(ln, decl, info_end)
        if rec.chrom != last:
            if rec.chrom in seen:
                raise UnsortedError(rec.chrom)
            seen.add(rec.chrom)
            last, last_pos = rec.chrom, -1
        if rec.pos < last_pos:
            raise UnsortedError(rec.pos)
        last_pos = rec.pos
        yield rec


def gvcf_to_bed_records(recs, gq_threshold: int = 20, gt: bool = True) -> tuple[list[tuple[str, int, int]], int]:
    """gvcf_to_bed's loop (gvcf_bed.py:38-68) over records: (the written intervals, the skipped count)."""
    out = []
    extent = -1
    last_chrom = ""
    skipped = 0
    for record in recs:
        if len(str(record.ref)) > 1 and (
            ("GQ" not in record.samples[0])
            or record.samples[0]["GT"] == (0, 0)
            or record.samples[0]["GT"] == (None, None)
        ):
            chrom, start, end = record.chrom, record.start, record.start + 1
        else:
            chrom, start, end = record.chrom, record.start, record.stop
        if chrom == last_chrom and start < extent:
            skipped += 1
            continue
        if chrom != last_chrom or extent < end:
            last_chrom = chrom
            extent = end
        if gt:
            if "GQ" in record.samples[0] and record.samples[0]["GQ"] >= gq_threshold:
                out.append((chrom, start, end))
        elif "GQ" not in record.samples[0] or record.samples[0]["GQ"] < gq_threshold:
            out.append((chrom, start, end))
    return out, skipped


def merge(intervals) -> list[tuple[str, int, int]]:
    """bedtools merge -d 0 of sorted intervals."""
    out: list[list] = []
    for c, s, e in intervals:
        if out and out[-1][0] == c and s <= out[-1][2]:
            out[-1][2] = max(out[-1][2], e)
        else:
            out.append([c, s, e])
    return [tuple(x) for x in out]


def bed_text(intervals) -> str:
    return "".join(f"{c}\t{s}\t{e}\n" for c, s, e in intervals)


ERROR_KINDS = ((LiteralError, "literal"), (UnsortedError, "unsorted"), (TypeError, "type"), (KeyError, "key"))


def run_text(text: str, gq_threshold: int = 20, gt: bool = True, do_merge: bool = False) -> dict:
    """The tool on VCF text: {"bed", "skipped"} or {"error": (record, kind)} where kind is "literal" / "unsorted" /
    "type" / "key" and record the 0-based data line it raises at."""
    count = [0]

    def counted():
        for rec in iterate(text):
            count[0] += 1
            yield rec

    try:
        ivs, skipped = gvcf_to_bed_records(counted(), gq_threshold, gt)
    except Exception as err:  # noqa: BLE001
        for cls, kind in ERROR_KINDS:
            if isinstance(err, cls):
                # a typing / order error is raised while the record is read (not yet counted)
                at = count[0] if cls in (LiteralError, UnsortedError) else count[0] - 1
                return {"error": (at, kind)}
        raise
    return {"bed": bed_text(merge(ivs) if do_merge else ivs), "skipped": skipped}
