"""calibrate_bridging_snvs -- H100-native drop-in for the reference tool.

Mirrors ``ugvc/pipelines/vcfbed/calibrate_bridging_snvs.py``: same flags and defaults (``init_parser``, :69-88), same
per-record rule (``is_homopolymer_snp`` :9-66 and ``run`` :91-130), same log lines of each rescued record, the header
unchanged and a bgzip'ed output with its ``.tbi`` (``pysam.tabix_index``, :130).

The work runs on the device (DESIGN.md 4d): the FASTA contigs are uploaded once per run, the input is cut into pieces of
whole lines, and each piece's compressed blocks (or plain text) go to the GPU, where they are inflated, indexed,
decided (the FASTA window walked in place), written with the new QUAL and FILTER columns and deflated again
(``ugvc_bsn_bgzf``); two pieces are in flight on two lanes.  The host cuts the pieces, appends the compressed blocks,
writes the index and the log lines.  There is no CPU path: without a device the tool raises.
"""
from __future__ import annotations

import argparse
import contextlib
import logging
import os

import numpy as np

from variantcalling_b200 import bgzf_io, lib, vcf_pieces
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.multiallelics import read_fasta_contig
from variantcalling_b200.vcf_header import VcfHeader

logger = logging.getLogger(__name__)

PIECE_BYTES = 64 << 20  # uncompressed text per device call
KEYS = ("AD", "DP", "BG_AD", "BG_DP")


def parse_args(argv: list[str]) -> argparse.Namespace:
    parser = argparse.ArgumentParser(prog="calibrate_bridging_snvs", description=run.__doc__)
    parser.add_argument("--vcf", required=True, help="Path to the VCF file")
    parser.add_argument("--reference", required=True, help="Path to the reference genome")
    parser.add_argument("--output", required=True, help="name of output vcf file")
    parser.add_argument("--min_query_hmer_size", default=5, type=int,
                        help="min size of the homopolymer in the query genome (with SNV alt allele) to be considered")
    parser.add_argument("--min_initial_qual", default=5, type=int, help="min quality of the initial SNV call")
    parser.add_argument("--min_tumor_vaf", default=0.2, type=float, help="min variant allele frequency in the tumor")
    parser.add_argument("--max_normal_vaf", default=0.1, type=float, help="max variant allele frequency in the normal")
    parser.add_argument("--min_normal_depth", default=10, type=int, help="min depth in the normal")
    parser.add_argument("--min_distance_from_edge", default=0, type=int, help="min distance from the edge of the homopolymer")
    parser.add_argument("--set_qual", default=20, type=int, help="set the quality of the SNV to this value")
    # host knob (not in the reference)
    parser.add_argument("--device", type=int, default=None, help="CUDA device index (default: LOCAL_RANK or 0)")
    return parser.parse_args(argv)


def qual_text(set_qual) -> bytes:
    """The QUAL column of a rescued record: htslib stores record.qual as float32 and prints it with %g (kputd)."""
    return ("%g" % float(np.float32(set_qual))).encode()


def bsn_params(header: VcfHeader, min_query_hmer_size=5, min_initial_qual=5, min_tumor_vaf=0.2, max_normal_vaf=0.1,
               min_normal_depth=10, min_distance_from_edge=0, set_qual=20):
    """The kernels' parameters: thresholds, the QUAL text and how the header types AD / DP / BG_AD / BG_DP.
    NotImplementedError for a rescue key of another Type than Integer / Float, ValueError for a negative
    min_query_hmer_size."""
    if int(min_query_hmer_size) < 0:
        raise ValueError(f"min_query_hmer_size {min_query_hmer_size} < 0: the FASTA window would end before it starts")
    kinds = []
    for key in KEYS:
        if key not in header.formats:
            kinds += [lib.BSN_KIND_NONE, 0]
            continue
        number, vtype = header.formats[key]
        if vtype not in ("Integer", "Float"):
            raise NotImplementedError(f"FORMAT/{key} of Type={vtype}: the rescue needs Integer or Float values")
        kinds += [lib.BSN_KIND_SCALAR if number == "1" else lib.BSN_KIND_TUPLE, int(vtype == "Integer")]
    q = qual_text(set_qual)
    if len(q) > lib.BSN_MAX_QUAL_BYTES:
        raise ValueError(f"set_qual {set_qual!r} prints as more than {lib.BSN_MAX_QUAL_BYTES} bytes")
    p = lib.BsnParams(int(min_query_hmer_size), int(min_distance_from_edge), float(min_initial_qual), float(min_tumor_vaf),
                      float(max_normal_vaf), float(min_normal_depth), q, len(q), *kinds)
    p._keep = q  # the bytes qual_text points into
    return p


def fasta_names(path: str) -> list[str]:
    """Contig names of a FASTA, from its .fai when present."""
    if os.path.exists(path + ".fai"):
        with open(path + ".fai") as fh:
            return [ln.split("\t", 1)[0] for ln in fh if ln.strip()]
    names = []
    with open(path, "rb") as fa:
        for ln in fa:
            if ln.startswith(b">") and ln[1:].split():
                names.append(ln[1:].split()[0].decode())
    return names


def load_contigs(reference: str, vcf: str) -> dict[str, bytes]:
    """Raw bytes of the contigs the run may read, each read once: those the input's .tbi names, else every FASTA
    contig.  A contig the FASTA lacks is left out (a record on it raises when it reaches the window)."""
    in_fasta = fasta_names(reference)
    wanted = in_fasta
    if os.path.exists(vcf + ".tbi"):
        try:
            names, _ = bgzf_io.read_tbi(vcf + ".tbi", linear=True)
            have = set(in_fasta)
            wanted = [c for c in names if c in have]
        except OSError:
            wanted = in_fasta
    if not os.path.exists(reference + ".fai"):  # one linear scan for all of them
        return _scan_fasta(reference, set(wanted))
    return {c: read_fasta_contig(reference, c, as_bytes=True) for c in dict.fromkeys(wanted)}


def _scan_fasta(path: str, wanted: set) -> dict[str, bytes]:
    out, name, parts = {}, None, []
    with open(path, "rb") as fa:
        for ln in fa:
            if ln.startswith(b">"):
                if name is not None and name not in out:
                    out[name] = b"".join(parts)
                toks = ln[1:].split()
                name = toks[0].decode() if toks and toks[0].decode() in wanted else None
                parts = []
            elif name is not None:
                parts.append(ln.strip())
    if name is not None and name not in out:
        out[name] = b"".join(parts)
    return out


def _raise_for(err: lib.UgvcDataError, rec: int, line: str, m: int):
    """The reference's exception for record `rec` (global index) whose device call reported err.bsn_reason."""
    cols = line.split("\t")
    where = f"record {rec} ({cols[0]}:{cols[1] if len(cols) > 1 else '?'})"
    reason = err.bsn_reason
    if reason == lib.BSN_E_TYPE:
        raise TypeError(f"{where}: None or a tuple where the rule needs a number (ALT '.', QUAL '.', a sliced scalar, "
                        f"or a missing AD / DP / BG_AD / BG_DP value)") from err
    if reason == lib.BSN_E_ZERO_DIVISION:
        raise ZeroDivisionError(f"{where}: DP is 0") from err
    if reason == lib.BSN_E_KEY:
        raise KeyError(f"{where}: invalid FORMAT: one of AD / DP / BG_AD / BG_DP is not in the header or the record") from err
    if reason == lib.BSN_E_FETCH:
        start = int(cols[1]) - m - 1
        if start < 0:
            raise ValueError(f"{where}: start out of range ({start})") from err
        raise ValueError(f"{where}: failure when retrieving sequence on '{cols[0]}'") from err
    raise lib.UgvcDataError(err.code, f"{where}: a QUAL / AD / DP / BG_AD / BG_DP literal that cannot be parsed") from err


def calibrate_bridging_snvs(
    vcf: str,
    reference: str,
    output: str,
    min_query_hmer_size: int = 5,
    min_initial_qual: int = 5,
    min_tumor_vaf: float = 0.2,
    max_normal_vaf: float = 0.1,
    min_normal_depth: int = 10,
    min_distance_from_edge: int = 0,
    set_qual: int = 20,
    device: int | None = None,
) -> int:
    """Un-filter the bridging SNVs of `vcf` into `output` (BGZF + .tbi; a name without .gz gets it).  Returns the
    rescued count."""
    header_text = bgzf_io.read_header_text(vcf)
    header = VcfHeader(header_text)
    params = bsn_params(header, min_query_hmer_size, min_initial_qual, min_tumor_vaf, max_normal_vaf, min_normal_depth,
                        min_distance_from_edge, set_qual)
    final = output if output.endswith(".gz") else output + ".gz"  # pysam.tabix_index compresses a plain file
    src = vcf_pieces.Input(vcf, len(header_text.encode()), PIECE_BYTES)
    pieces = src.pieces
    contigs = load_contigs(reference, vcf)

    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    ctx = lib.Context(device)
    log_records = logger.isEnabledFor(logging.INFO)
    try:
        for name, seq in contigs.items():
            ctx.bsn_add_contig(name, seq)
        ctx.load_plan(MC.compile_plan_no_model(header).blob)
        cap = max([p[3] for p in pieces], default=1) + 64
        ctx.reserve(cap, cap // 8 + 16, 2 if len(pieces) > 1 else 1)

        def one(k: int, lane: int):
            data, skip, take, _span = pieces[k]
            return ctx.bsn_bgzf(data, skip, take, not src.is_bgzf, params, cap // 8 + 16, lane=lane)

        writer = bgzf_io.BgzfWriter(final)
        # the header as htslib writes it back: unchanged, with the PASS line it always carries
        writer.write(("\n".join(header.edited_lines(with_model=False, with_blacklist=False)) + "\n").encode())
        index = vcf_pieces.Index("END" in header.info)
        n_rescued = 0
        first = 0  # records of the pieces written so far
        done = 0
        try:
            with contextlib.closing(vcf_pieces.run_on_lanes(ctx, len(pieces), one, "ugvc-bsn")) as results:
                for k, res in results:
                    base = writer.uoffset
                    writer.write_compressed(res["bgzf"], res["block_csize"], int(res["line_start"][-1]), lib.DEF_CHUNK)
                    index.add(writer, res, base)
                    if log_records and res["n_rescued"]:
                        _log_rescued(src, src.starts[k], res, contigs, params.min_query_hmer_size)
                    n_rescued += res["n_rescued"]
                    first += res["n_records"]
                    done += 1
                    pieces[k] = None
        except lib.UgvcDataError as err:
            if getattr(err, "bsn_record", -1) < 0:
                raise
            line = src.line_at(src.starts[done], err.bsn_record)
            _raise_for(err, first + err.bsn_record, line, params.min_query_hmer_size)
        writer.close()
        index.write(final + ".tbi")
    finally:
        ctx.close()
    return n_rescued


def _log_rescued(src: vcf_pieces.Input, u0: int, res: dict, contigs: dict, m: int):
    """The reference's two log lines of each rescued record: its FASTA window and hmer_size, then the record as read
    (pysam's str(record) ends with the newline)."""
    sl = res["src_line_start"]
    for r in np.flatnonzero(res["flags"] & lib.BSN_RESCUED).tolist():
        line = src.text(u0 + int(sl[r]), u0 + int(sl[r + 1])).decode("latin-1")
        cols = line.split("\t", 2)
        pos = int(cols[1])
        seq = contigs[cols[0]][pos - m - 1: pos + m].decode("latin-1")
        logger.info(f"refseq : {seq} hmer_size: {int(res['hmer'][r])}")
        logger.info(line)


def run(argv: list[str]):
    """
    Un-filter SNVs which generate a long homopolymer, have borderline quality
    and have a high VAF in the tumor and low VAF in the normal
    * DV often filters such true SNVs due to low confidence of the allele (SNV / deletion)
    """
    logging.basicConfig(format="%(asctime)s %(message)s", level=logging.INFO)
    args = parse_args(argv)
    calibrate_bridging_snvs(
        vcf=args.vcf,
        reference=args.reference,
        output=args.output,
        min_query_hmer_size=args.min_query_hmer_size,
        min_initial_qual=args.min_initial_qual,
        min_tumor_vaf=args.min_tumor_vaf,
        max_normal_vaf=args.max_normal_vaf,
        min_normal_depth=args.min_normal_depth,
        min_distance_from_edge=args.min_distance_from_edge,
        set_qual=args.set_qual,
        device=args.device,
    )


def main():
    import sys

    run(sys.argv[1:])


if __name__ == "__main__":
    main()
