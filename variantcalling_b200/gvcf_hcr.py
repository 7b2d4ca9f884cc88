"""gvcf_hcr -- H100-native drop-in for the reference tool.

Mirrors ``ugvc/joint/gvcf_bed.py:gvcf_to_bed`` (same signature and return value: the skipped count) and
``ugvc/pipelines/vcfbed/gvcf_hcr_main.py`` (same flags and log lines; ``gvcf_to_bed(gt=True)`` then ``bedtools merge``,
whose default ``-d 0`` joins book-ended intervals).  No step-1 file is made: the merged BED is written directly.

The work runs on the device (DESIGN.md 4e): the input is cut into pieces of whole lines, each piece's compressed blocks
go to the GPU, where they are inflated, indexed and decided, and the per-contig prefix maximum of the interval ends is
taken (``ugvc_hcr_scan``, two pieces in flight on two lanes).  Whether a record is kept depends on the end of the last
kept record before it, so the second half (``ugvc_hcr_emit``: kept flags, selection, merge marks, the BED text) runs in
piece order with the previous piece's exit state.  The host cuts the pieces, names the contig runs, joins the last
merged interval of a piece with the first of the next and writes the text.  There is no CPU path: without a device the
tool raises.
"""
from __future__ import annotations

import argparse
import contextlib
import logging
import os
import threading

from variantcalling_b200 import bgzf_io, lib, vcf_pieces
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader

logger = logging.getLogger(__name__)

PIECE_BYTES = 64 << 20  # uncompressed text per device call


def parse_args(argv: list[str]) -> argparse.Namespace:
    parser = argparse.ArgumentParser(prog="gvcf_hcr", description="Extract bed of high confidence regions from a gvcf file.")
    parser.add_argument("--gvcf", type=str, required=True, help="Path to the gvcf file.")
    parser.add_argument("--bed", type=str, required=True, help="Path to the output bed file.")
    parser.add_argument("--gq_threshold", type=int, default=20, help="GQ threshold.")
    # host knob (not in the reference)
    parser.add_argument("--device", type=int, default=None, help="CUDA device index (default: LOCAL_RANK or 0)")
    return parser.parse_args(argv)


def hcr_params(header: VcfHeader, gq_threshold: int = 20, gt: bool = True, merge: bool = False) -> lib.HcrParams:
    """The kernels' parameters: the threshold, the mode, whether INFO/END sets intervals and how the header types GQ
    (undeclared keys are typed String by htslib)."""
    kind, integer = lib.HCR_GQ_STRING, 0
    if "GQ" in header.formats:
        number, vtype = header.formats["GQ"]
        if vtype in ("Integer", "Float"):
            kind = lib.HCR_GQ_SCALAR if number == "1" else lib.HCR_GQ_TUPLE
            integer = int(vtype == "Integer")
    return lib.HcrParams(int(gq_threshold), int(bool(gt)), int(bool(merge)), int("END" in header.info), kind, integer)


def _raise_for(reason: int, rec: int, line: str, err: Exception | None):
    """The reference's exception for record `rec` (global index)."""
    cols = line.split("\t")
    where = f"record {rec} ({cols[0]}:{cols[1] if len(cols) > 1 else '?'})"
    if reason == lib.HCR_E_TYPE:
        raise TypeError(f"{where}: GQ is None, a tuple or a string where it is compared with the threshold") from err
    if reason == lib.HCR_E_KEY:
        raise KeyError(f"{where}: invalid FORMAT: GT (a RefCall deletion candidate with GQ but no GT)") from err
    if reason == lib.HCR_E_UNSORTED:
        raise ValueError(f"{where}: records are not sorted by contig and position: the file cannot be indexed") from err
    raise lib.UgvcDataError(lib.UGVC_E_DATA, f"{where}: a GQ / GT literal that cannot be parsed") from err


def join_pieces(held: bytes, bed: bytes) -> tuple[bytes, bytes]:
    """Merged BED text across pieces: given the last line so far (held back, b"" when none) and the next piece's merged
    lines, (the text to write now, the new last line).  The piece's first line extends the held one when it is on the
    same chrom and starts at or before its end (bedtools merge -d 0)."""
    if not bed:
        return b"", held
    out = b""
    if held:
        nl = bed.index(b"\n") + 1
        c0, s0, e0 = held.rstrip(b"\n").split(b"\t")
        c1, s1, e1 = bed[:nl].rstrip(b"\n").split(b"\t")
        if c0 == c1 and int(s1) <= int(e0):
            held = b"\t".join((c0, s0, e1)) + b"\n"
            bed = bed[nl:]
        if not bed:
            return b"", held
        out = held
    cut = bed.rindex(b"\n", 0, len(bed) - 1) + 1 if bed.count(b"\n") > 1 else 0
    return out + bed[:cut], bed[cut:]


class _Failed(Exception):
    """An earlier piece failed: this one is not emitted (the earlier piece's exception is raised first)."""


def _lines(gvcf: str, gq_threshold: int, gt: bool, merge: bool, device: int | None, write) -> int:
    """BED text of `gvcf` handed to write() in file order (merged lines joined across pieces); returns the skipped
    count."""
    if not (os.path.exists(gvcf + ".tbi") or os.path.exists(gvcf + ".csi")):
        raise ValueError(f"fetch requires an index: {gvcf} has no .tbi / .csi")
    with open(gvcf, "rb") as fh:
        if fh.read(2) != b"\x1f\x8b":
            raise ValueError(f"fetch requires an index: {gvcf} is not BGZF-compressed")
    header_text = bgzf_io.read_header_text(gvcf)
    header = VcfHeader(header_text)
    params = hcr_params(header, gq_threshold, gt, merge)
    src = vcf_pieces.Input(gvcf, len(header_text.encode()), PIECE_BYTES, index_cuts=False)
    pieces = src.pieces
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    ctx = lib.Context(device)
    # piece k's exit state, published for piece k + 1: (last contig, exit extent, POS - 1 of the last record, records
    # so far, contigs seen), or None when piece k failed
    states: dict[int, tuple | None] = {-1: (None, -1, -1, 0, frozenset())}
    cond = threading.Condition()

    def publish(k: int, state):
        with cond:
            states[k] = state
            cond.notify_all()

    def one(k: int, lane: int):
        try:
            data, skip, take, span = pieces[k]
            sc = ctx.hcr_scan(data, skip, take, params, cap // 8 + 16, lane=lane)
            n = sc["n_records"]
            names = [src.text(src.starts[k] + int(a), src.starts[k] + int(a) + 4096).split(b"\t", 1)[0].decode()
                     for _, a in sc["runs"]]
            with cond:
                cond.wait_for(lambda: k - 1 in states)
                prev = states[k - 1]
            if prev is None:
                raise _Failed
            last_chrom, extent, last_start, first, seen = prev
            cont = n > 0 and names[0] == last_chrom
            # the first record where the host sees a file that cannot be indexed
            bad = n if not (cont and sc["first_start"] < last_start) else 0
            seen_here = set(seen)
            for (r, _), name in zip(sc["runs"], names):
                if (r > 0 or not cont) and name in seen_here:
                    bad = min(bad, int(r))
                seen_here.add(name)
            try:
                em = ctx.hcr_emit(params, cont, extent, span + 48 * n + 64, lane=lane)
            except lib.UgvcDataError as err:
                if getattr(err, "hcr_record", -1) < 0:
                    raise
                r = err.hcr_record
                if bad < r or (bad == r and err.hcr_reason != lib.HCR_E_LITERAL):
                    r, reason = bad, lib.HCR_E_UNSORTED
                else:
                    reason = err.hcr_reason
                _raise_for(reason, first + r, src.line_at(src.starts[k], r), err)
            if bad < n:
                _raise_for(lib.HCR_E_UNSORTED, first + bad, src.line_at(src.starts[k], bad), None)
            publish(k, (names[-1] if names else last_chrom, em["exit_extent"], sc["last_start"] if n else last_start,
                        first + n, frozenset(seen_here)))
            return em
        except BaseException:
            publish(k, None)
            raise

    skipped = 0
    try:
        ctx.load_plan(MC.compile_plan_no_model(header).blob)
        cap = max([p[3] for p in pieces], default=1) + 64
        ctx.reserve(cap, cap // 8 + 16, 2 if len(pieces) > 1 else 1)
        held = b""  # merging: the last line so far, which the next piece's first line may extend
        with contextlib.closing(vcf_pieces.run_on_lanes(ctx, len(pieces), one, "ugvc-hcr")) as results:
            for k, em in results:
                skipped += em["skipped"]
                bed = em["bed"]
                pieces[k] = None
                if not merge:
                    write(bed)
                    continue
                now, held = join_pieces(held, bed)
                write(now)
        if held:
            write(held)
    finally:
        ctx.close()
    return skipped


def gvcf_to_bed(gvcf_file: str, bed_file: str, gq_threshold: int = 20, gt: bool = True, device: int | None = None) -> int:
    """Select records with GQ >= (gt=True) or < (gt=False, or GQ absent) gq_threshold among the records that are not
    skipped, and write their intervals to a BED file.  Returns the number of skipped records."""
    with open(bed_file, "wb") as out:
        return _lines(gvcf_file, gq_threshold, gt, False, device, out.write)


def gvcf_hcr(gvcf: str, bed: str, gq_threshold: int = 20, device: int | None = None) -> None:
    """The BED of the high-confidence regions of `gvcf`: gvcf_to_bed(gt=True) with book-ended intervals merged."""
    with open(bed, "wb") as out:
        _lines(gvcf, gq_threshold, True, True, device, out.write)


def run(argv: list[str]):
    """Converts gVCF to high confidence BED file."""
    logging.basicConfig(format="%(asctime)s %(message)s", level=logging.INFO)
    args = parse_args(argv)
    logger.info("Step 1: Create intervals of high confidence")
    logger.info("Step 2: Merge intervals")
    gvcf_hcr(args.gvcf, args.bed, args.gq_threshold, device=args.device)


def main():
    import sys

    run(sys.argv[1:])


if __name__ == "__main__":
    main()
