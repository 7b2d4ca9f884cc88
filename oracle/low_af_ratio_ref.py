"""ORACLE (test infrastructure, not product code).

filter_low_af_ratio_to_background (``ugbio_filtering/filter_low_af_ratio_to_background.py``) restated over text, for the
tests of the device path (DESIGN.md 4c):

* every sample's GT / VAF / BG_VAF typed as ``oracle/vcf_reader.py`` types the first sample (``typed_value`` /
  ``parse_gt``), with an undeclared VAF / BG_VAF as None, and a literal those refuse raising :class:`LiteralError`;
* ``process_record`` (:75-114) over those typed samples, ``failed`` carried from sample to sample;
* the FILTER edit of pysam's ``record.filter.clear()`` / ``add()`` -- htslib's ``bcf_add_filter``: adding skips an ID
  already present, ``PASS`` replaces the list, anything added to ``[PASS]`` replaces it, an empty list prints ``.``;
* the expected output text, and the interval of every record in the output's tabix index.

``tests/golden/low_af_ratio.json.gz`` (scripts/make_golden_low_af_ratio.py) pins the decision to the reference's own
``process_record``; the FILTER edit is htslib's and parity-unpinned here (no pysam), so every case is crafted.
"""
from __future__ import annotations

from oracle.vcf_reader import OracleHeader, parse_gt, typed_value

DEFAULT_FILTER = "LowAFRatioToBackground"


class LiteralError(ValueError):
    """A GT / VAF / BG_VAF literal that cannot be typed (the product raises UgvcDataError for the record)."""


def filter_description(af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold) -> str:
    return (f"Filter variants if AF ratio to background in GT ALT alleles < threshold. "
            f"For snps and non-h-indels: {af_ratio_threshold}, and "
            f"for h-indels (applied only if tumor VAF<{t_vaf_threshold}: {af_ratio_threshold_h_indels})")


def header_kinds(header: OracleHeader) -> dict:
    """How the header types the three tags: {"VARIANT_TYPE": compares with "h-indel", "VAF"/"BG_VAF": (Number, Type) or
    None}.  NotImplementedError for a VAF / BG_VAF of another Type than Float / Integer."""
    n, t = header.info.get("VARIANT_TYPE", (".", "String"))
    out = {"VARIANT_TYPE": "VARIANT_TYPE" in header.info and n == "1" and t in ("String", "Character")}
    for key in ("VAF", "BG_VAF"):
        if key not in header.formats:
            out[key] = None
            continue
        number, vtype = header.formats[key]
        if vtype not in ("Float", "Integer"):
            raise NotImplementedError(f"FORMAT/{key} of Type={vtype}")
        out[key] = (number, vtype)
    return out


def _typed(text, decl):
    number, vtype = decl
    if text is None or text == ".":
        return None if number == "1" else (None,)
    try:
        return typed_value(text, number, vtype)
    except ValueError as err:
        raise LiteralError(text) from err


def typed_samples(line: str, kinds: dict) -> list[dict]:
    """{"GT", "VAF", "BG_VAF"} of every sample column (a key the FORMAT does not carry is absent)."""
    cols = line.rstrip("\n").split("\t")
    if len(cols) <= 9 or cols[8] == ".":  # noqa: PLR2004
        return [{} for _ in cols[9:]]
    keys = cols[8].split(":")
    out = []
    for sample in cols[9:]:
        vals = sample.split(":")
        d = {}
        for i, key in enumerate(keys):
            text = vals[i] if i < len(vals) else None
            if key == "GT":
                try:
                    d[key] = parse_gt(text if text is not None else ".")
                except ValueError as err:
                    raise LiteralError(text) from err
            elif key in ("VAF", "BG_VAF") and kinds[key] is not None:
                d[key] = _typed(text, kinds[key])
        out.append(d)
    return out


def process_record(samples: list[dict], af_ratio_threshold, t_vaf_threshold) -> bool:
    """The reference's process_record (:75-114) over typed samples; len() of a scalar raises TypeError as there."""
    failed = False
    for s in samples:
        gt, vaf, bg_vaf = s.get("GT"), s.get("VAF"), s.get("BG_VAF")
        if gt is None or vaf is None or bg_vaf is None:
            continue
        for allele in gt:
            if allele is None or allele == 0:
                continue
            if allele - 1 >= len(vaf) or allele - 1 >= len(bg_vaf):
                continue
            if vaf[allele - 1] is None or vaf[allele - 1] == 0:
                failed = True
                continue
            if bg_vaf[allele - 1] is None or bg_vaf[allele - 1] == 0:
                failed = False
                break
            if vaf[allele - 1] / bg_vaf[allele - 1] >= af_ratio_threshold or vaf[allele - 1] >= t_vaf_threshold:
                failed = False
                break
            failed = True
    return failed


def add_filter(flt: list[str], fid: str) -> list[str]:
    """htslib bcf_add_filter on a list of IDs."""
    if fid in flt:
        return flt
    if fid == "PASS" or flt == ["PASS"]:
        return [fid]
    return [*flt, fid]


def edit_record(line: str, kinds: dict, af_ratio_threshold=10, af_ratio_threshold_h_indels=0, t_vaf_threshold=0,
                new_filter: str = DEFAULT_FILTER) -> tuple[str, bool]:
    """(output line, failed) of one data line (no newline).  Raises LiteralError / TypeError as described above."""
    cols = line.split("\t")
    samples = typed_samples(line, kinds)  # every literal is typed when the record is read
    ids = [] if cols[6] == "." else cols[6].split(";")
    if "RefCall" in ids:
        return line, False
    vt = None
    if cols[7] != ".":
        for kv in cols[7].split(";"):
            key, sep, val = kv.partition("=")
            if key == "VARIANT_TYPE":
                vt = (val or None) if sep else None
    h_indel = kinds["VARIANT_TYPE"] and vt == "h-indel"
    thr = af_ratio_threshold_h_indels if h_indel else af_ratio_threshold
    vthr = t_vaf_threshold if h_indel else 1
    failed = process_record(samples, thr, vthr)
    rebuilt = new_filter in ids
    flt = ids
    if rebuilt:
        flt = []
        for f in ids:
            if f != new_filter:
                flt = add_filter(flt, f)
    if failed:
        flt = add_filter(flt, new_filter)
    if rebuilt or failed:
        cols[6] = ";".join(flt) if flt else "."
    return "\t".join(cols), failed


def run_text(text: str, af_ratio_threshold=10, af_ratio_threshold_h_indels=0, t_vaf_threshold=0,
             new_filter: str = DEFAULT_FILTER) -> dict:
    """The whole tool on VCF text: {"header", "records", "failed", "n_filtered"} or {"error": (record, kind)} where kind is
    "literal" / "type" and record the 0-based data line it raises at."""
    lines = text.split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    head = [ln for ln in lines if ln.startswith("#")]
    data = [ln for ln in lines if ln and not ln.startswith("#")]
    header = OracleHeader(head)
    kinds = header_kinds(header)
    out_head = list(head)
    if new_filter not in header.filters:
        desc = filter_description(af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold)
        at = next(i for i, ln in enumerate(out_head) if ln.startswith("#CHROM"))
        out_head.insert(at, f'##FILTER=<ID={new_filter},Description="{desc}">')
    if not any(ln.startswith("##FILTER=<ID=PASS,") for ln in out_head):
        out_head.insert(1 if out_head and out_head[0].startswith("##fileformat") else 0,
                        '##FILTER=<ID=PASS,Description="All filters passed">')
    records, failed = [], []
    for i, ln in enumerate(data):
        try:
            r, f = edit_record(ln, kinds, af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold, new_filter)
        except LiteralError:
            return {"error": (i, "literal")}
        except TypeError:
            return {"error": (i, "type")}
        records.append(r)
        failed.append(f)
    return {"header": out_head, "records": records, "failed": failed, "n_filtered": sum(failed)}


def intervals(records: list[str], info_end: bool) -> list[tuple[str, int, int]]:
    """(contig, beg, end) of every record in the output's tabix index: POS - 1 to POS - 1 + len(REF), or INFO/END when
    the header declares it and the first END= field is digits beyond POS - 1."""
    out = []
    for ln in records:
        cols = ln.split("\t")
        beg = int(cols[1]) - 1
        end = beg + max(1, len(cols[3]))
        if info_end and cols[7] != ".":
            for kv in cols[7].split(";"):
                if kv.startswith("END="):
                    v = kv[4:]
                    if v.isdigit() and 0 < len(v) <= 10 and int(v) > beg:  # noqa: PLR2004
                        end = int(v)
                    break
        out.append((cols[0], beg, end))
    return out
