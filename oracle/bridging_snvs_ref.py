"""ORACLE (test infrastructure, not product code).

calibrate_bridging_snvs (``ugvc/pipelines/vcfbed/calibrate_bridging_snvs.py``) restated over text, for the tests of the
device path (DESIGN.md 4d):

* the candidate test of ``is_homopolymer_snp`` (:16-22) on the line's REF / ALT / FILTER / QUAL, short-circuit as there;
* the FASTA window ``fetch(chrom, pos - m - 1, pos + m)`` as a slice of the contig's raw bytes (pysam's ``ValueError`` for a
  negative start or a contig the FASTA lacks), the two walks and the qualifying test (:26-62);
* the rescue of ``run`` (:96-103) on sample 0's AD / DP / BG_AD / BG_DP, typed as ``oracle/vcf_reader.py`` types values
  (Number=1 a scalar, any other Number a tuple, ``.`` or a dropped sub-field None / (None,)), in Python's order of
  evaluation, raising what Python raises;
* the edit (QUAL = ``"%g" % float32(set_qual)``, FILTER = ``PASS``) and the log lines of each rescued record.

``tests/golden/bridging_snvs.json.gz`` (scripts/make_golden_bridging_snvs.py) pins all of it to the reference's own
``run`` and ``is_homopolymer_snp``.
"""
from __future__ import annotations

import re

import numpy as np

from oracle.vcf_reader import OracleHeader

KEYS = ("AD", "DP", "BG_AD", "BG_DP")
_INT = re.compile(r"[+-]?[0-9]{1,18}")
_FLOAT = re.compile(r"[+-]?([0-9]+\.?[0-9]*([eE][+-]?[0-9]+)?|\.[0-9]+([eE][+-]?[0-9]+)?|nan|inf|infinity)", re.IGNORECASE)


class LiteralError(ValueError):
    """A QUAL / rescue-key literal that cannot be typed (the product raises UgvcDataError for the record)."""


class FetchError(ValueError):
    """pysam FastaFile.fetch's ValueError: a negative window start or a contig the FASTA does not hold."""


def qual_text(set_qual) -> str:
    """The QUAL column of a rescued record: htslib stores float32 and prints it with %g."""
    return "%g" % float(np.float32(set_qual))


def header_kinds(header: OracleHeader) -> dict:
    """(Number, Type) of each rescue key, None when undeclared.  NotImplementedError for a Type other than Integer /
    Float."""
    out = {}
    for key in KEYS:
        if key not in header.formats:
            out[key] = None
            continue
        number, vtype = header.formats[key]
        if vtype not in ("Integer", "Float"):
            raise NotImplementedError(f"FORMAT/{key} of Type={vtype}")
        out[key] = (number, vtype)
    return out


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


def _typed(text: str | None, decl):
    number, vtype = decl
    if text is None or text == ".":
        return None if number == "1" else (None,)
    if text == "":
        return None if number == "1" else ()
    if number == "1":
        return _elem(text, vtype)
    return tuple(_elem(t, vtype) for t in text.split(","))


def typed_sample0(cols: list[str], kinds: dict) -> dict:
    """The declared rescue keys sample 0 carries, typed; a key missing from the FORMAT column (or with no sample
    column) is absent."""
    if len(cols) <= 9 or cols[8] == ".":  # noqa: PLR2004
        return {}
    keys = cols[8].split(":")
    vals = cols[9].split(":")
    out = {}
    for i, key in enumerate(keys):
        if key in KEYS and kinds[key] is not None:
            out[key] = _typed(vals[i] if i < len(vals) else None, kinds[key])
    return out


def parse_qual(text: str):
    if text == ".":
        return None
    if not _FLOAT.fullmatch(text):
        raise LiteralError(text)
    return float(np.float32(float(text)))


def fetch(fasta: dict, chrom: str, start: int, end: int) -> bytes:
    if start < 0:
        raise FetchError(f"start out of range ({start})")
    if chrom not in fasta:
        raise FetchError(f"failure when retrieving sequence on '{chrom}'")
    return fasta[chrom][start:end]


def decide(line: str, kinds: dict, fasta: dict, m: int = 5, min_initial_qual=5, min_tumor_vaf=0.2, max_normal_vaf=0.1,
           min_normal_depth=10, min_distance_from_edge=0) -> tuple[bool, int, str | None]:
    """(rescued, hmer_size of a walked window else 0, the window text) of one data line.  Raises LiteralError,
    TypeError, ZeroDivisionError, KeyError or FetchError as described above."""
    cols = line.split("\t")
    qual = parse_qual(cols[5])
    s0 = typed_sample0(cols, kinds)  # every literal is typed when the record is read
    ref, alt_col = cols[3], cols[4]
    alts = None if alt_col == "." else alt_col.split(",")
    filters = [] if cols[6] == "." else cols[6].split(";")
    if not (len(ref) == 1 and len(alts) == 1 and len(alts[0]) == 1 and "PASS" not in filters and qual >= min_initial_qual):
        return False, 0, None
    alt = alts[0].encode()[0]
    pos = int(cols[1])
    seq = fetch(fasta, cols[0], pos - m - 1, pos + m)
    up = down = 0
    before = after = None
    for b in seq[m + 1:]:
        if b != alt:
            after = b
            break
        down += 1
    for b in seq[m - 1::-1]:
        if b != alt:
            before = b
            break
        up += 1
    hmer = 1 + up + down
    tandem = before is not None and before == after and chr(before) == ref and up == down
    text = seq.decode("latin-1")
    if not (hmer >= m and not tandem and min(up, down) >= min_distance_from_edge):
        return False, hmer, text
    normal_depth = s0["BG_DP"]
    tumor_vaf = sum(s0["AD"][1:]) / s0["DP"]
    normal_vaf = sum(s0["BG_AD"][1:]) / max(0.01, normal_depth)
    rescued = tumor_vaf >= min_tumor_vaf and normal_vaf <= max_normal_vaf and normal_depth > min_normal_depth
    return bool(rescued), hmer, text


ERROR_KINDS = ((LiteralError, "literal"), (FetchError, "fetch"), (TypeError, "type"), (ZeroDivisionError, "zero"),
               (KeyError, "key"))


def run_text(text: str, fasta: dict, min_query_hmer_size=5, min_initial_qual=5, min_tumor_vaf=0.2, max_normal_vaf=0.1,
             min_normal_depth=10, min_distance_from_edge=0, set_qual=20) -> dict:
    """The whole tool on VCF text: {"header", "records", "rescued", "hmer", "logs", "n_rescued"} or {"error": (record,
    kind)} where kind is "literal" / "fetch" / "type" / "zero" / "key" and record the 0-based data line it raises at."""
    lines = text.split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    head = [ln for ln in lines if ln.startswith("#")]
    data = [ln for ln in lines if ln and not ln.startswith("#")]
    kinds = header_kinds(OracleHeader(head))
    out_head = list(head)
    if not any(ln.startswith("##FILTER=<ID=PASS,") for ln in out_head):  # htslib always writes the PASS line
        out_head.insert(1 if out_head and out_head[0].startswith("##fileformat") else 0,
                        '##FILTER=<ID=PASS,Description="All filters passed">')
    qt = qual_text(set_qual)
    records, rescued, hmers, logs = [], [], [], []
    for i, ln in enumerate(data):
        try:
            r, h, seq = decide(ln, kinds, fasta, min_query_hmer_size, min_initial_qual, min_tumor_vaf, max_normal_vaf,
                               min_normal_depth, min_distance_from_edge)
        except Exception as err:  # noqa: BLE001
            for cls, kind in ERROR_KINDS:
                if isinstance(err, cls):
                    return {"error": (i, kind)}
            raise
        if r:
            logs += [f"refseq : {seq} hmer_size: {h}", ln + "\n"]
            cols = ln.split("\t")
            cols[5], cols[6] = qt, "PASS"
            ln = "\t".join(cols)
        records.append(ln)
        rescued.append(r)
        hmers.append(h)
    return {"header": out_head, "records": records, "rescued": rescued, "hmer": hmers, "logs": logs, "n_rescued": sum(rescued)}
