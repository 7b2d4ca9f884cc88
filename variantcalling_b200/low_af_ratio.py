"""filter_low_af_ratio_to_background -- H100-native drop-in for the reference tool.

Mirrors ``ugbio_filtering/filter_low_af_ratio_to_background.py``: same flags (``main``, :117-153), same function and
signature (:8-15), same header edit (:18-30), same log lines, same per-record rule (:35-65, ``process_record`` :75-114)
and a bgzip'ed output with its ``.tbi`` (``pysam.tabix_index``, :70).

The work runs on the device (DESIGN.md 4c): the input is cut into pieces of whole lines, each piece's compressed blocks
(or plain text) go to the GPU, where they are inflated, indexed, decided over every sample, written with the new FILTER
column and deflated again (``ugvc_afr_bgzf``); two pieces are in flight on two lanes.  The host only cuts the pieces,
appends the compressed blocks and writes the index.  There is no CPU path: without a device the tool raises.
"""
from __future__ import annotations

import argparse
import contextlib
import logging
import os

from variantcalling_b200 import bgzf_io, lib, vcf_pieces
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader

logger = logging.getLogger(__name__)

PIECE_BYTES = 64 << 20  # uncompressed text per device call
_BAD_ID_CHARS = set(";=,<>\"") | set(" \t\r\n\v\f")


def parse_args(argv: list[str]) -> argparse.Namespace:
    parser = argparse.ArgumentParser(description="Annotate variants with low AF ratio")
    parser.add_argument("input_vcf", help="Input VCF file")
    parser.add_argument("output_vcf", help="Output VCF file")
    parser.add_argument("--af_ratio_threshold", type=float, default=10,
                        help="AF ratio threshold for snps and non-h-indels (default: 10)")
    parser.add_argument("--tumor_vaf_threshold_h_indels", type=float, default=0,
                        help="Tumor VAF threshold for filtering (default: 0) - any h-indel with VAF above this threshold will "
                             "not be filtered")
    parser.add_argument("--af_ratio_threshold_h_indels", type=float, default=0,
                        help="AF ratio threshold for h-indels (default: 0)")
    parser.add_argument("--new_filter", default="LowAFRatioToBackground",
                        help="Name of new FILTER tag (default: LowAFRatioToBackground)")
    # host knob (not in the reference)
    parser.add_argument("--device", type=int, default=None, help="CUDA device index (default: LOCAL_RANK or 0)")
    return parser.parse_args(argv)


def filter_description(af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold) -> str:
    """The reference's description f-string (:25-29), from the values as passed."""
    return (f"Filter variants if AF ratio to background in GT ALT alleles < threshold. "
            f"For snps and non-h-indels: {af_ratio_threshold}, and "
            f"for h-indels (applied only if tumor VAF<{t_vaf_threshold}: {af_ratio_threshold_h_indels})")


def check_filter_id(new_filter: str):
    """A FILTER ID the output can carry; the reference hands any string to htslib (DESIGN.md 4c lists this deviation)."""
    raw = new_filter.encode()
    if (not raw or len(raw) > lib.AFR_MAX_FILTER_BYTES or new_filter in ("PASS", "RefCall")
            or any(c in _BAD_ID_CHARS for c in new_filter)):
        raise ValueError(f"new_filter {new_filter!r} is not a valid FILTER ID (1..{lib.AFR_MAX_FILTER_BYTES} bytes, none of "
                         f"';=,<>\"' or white space, not PASS / RefCall)")


def afr_params(header: VcfHeader, af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold, new_filter: str):
    """The kernels' parameters: thresholds, the FILTER ID and how the header types VARIANT_TYPE / VAF / BG_VAF.
    NotImplementedError for a VAF / BG_VAF of another Type than Float / Integer."""
    kinds = []
    for key in ("VAF", "BG_VAF"):
        if key not in header.formats:
            kinds += [lib.AFR_KIND_NONE, 0]
            continue
        number, vtype = header.formats[key]
        if vtype not in ("Float", "Integer"):
            raise NotImplementedError(f"FORMAT/{key} of Type={vtype}: the AF-ratio rule needs Float or Integer values")
        kinds += [lib.AFR_KIND_SCALAR if number == "1" else lib.AFR_KIND_TUPLE, int(vtype == "Integer")]
    vt = header.info.get("VARIANT_TYPE")
    vt_kind = int(vt is not None and vt[0] == "1" and vt[1] in ("String", "Character"))
    nf = new_filter.encode()
    p = lib.AfrParams(float(af_ratio_threshold), float(af_ratio_threshold_h_indels), float(t_vaf_threshold), nf, len(nf), vt_kind,
                      *kinds)
    p._keep = nf  # the bytes new_filter points into
    return p


def output_lines(header: VcfHeader, new_filter: str, desc: str) -> list[str]:
    """Header of the output: the FILTER line added before #CHROM unless declared, PASS as VcfHeader.edited_lines has it."""
    lines = header.edited_lines(with_model=False, with_blacklist=False)
    if new_filter in header.filters:
        logger.warning(f"Existing {new_filter} filter found in header. It will be replaced.")
        return lines
    at = next(i for i, ln in enumerate(lines) if ln.startswith("#CHROM"))
    return lines[:at] + [f'##FILTER=<ID={new_filter},Description="{desc}">'] + lines[at:]


def filter_low_af_ratio_to_background(
    input_vcf: str,
    output_vcf: str,
    af_ratio_threshold: float = 10,
    af_ratio_threshold_h_indels: float = 0,
    t_vaf_threshold: float = 0,
    new_filter: str = "LowAFRatioToBackground",
    device: int | None = None,
):
    check_filter_id(new_filter)
    header_text = bgzf_io.read_header_text(input_vcf)
    header = VcfHeader(header_text)
    params = afr_params(header, af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold, new_filter)
    desc = filter_description(af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold)
    lines = output_lines(header, new_filter, desc)
    final = output_vcf if output_vcf.endswith(".gz") else output_vcf + ".gz"  # pysam.tabix_index compresses a plain file
    src = vcf_pieces.Input(input_vcf, len(header_text.encode()), PIECE_BYTES)
    pieces = src.pieces

    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    ctx = lib.Context(device)
    ctx.load_plan(MC.compile_plan_no_model(header).blob)
    cap = max([p[3] for p in pieces], default=1) + 64
    ctx.reserve(cap, cap // 8 + 16, 2 if len(pieces) > 1 else 1)

    logger.info(f"Processing {input_vcf} and writing to {output_vcf}")

    def one(k: int, lane: int):
        data, skip, take, _span = pieces[k]
        return ctx.afr_bgzf(data, skip, take, not src.is_bgzf, params, cap // 8 + 16, lane=lane)

    writer = bgzf_io.BgzfWriter(final)
    writer.write(("\n".join(lines) + "\n").encode())
    index = vcf_pieces.Index("END" in header.info)
    filtered_count = 0
    first = 0
    try:
        try:
            with contextlib.closing(vcf_pieces.run_on_lanes(ctx, len(pieces), one, "ugvc-afr")) as results:
                for k, res in results:
                    base = writer.uoffset
                    writer.write_compressed(res["bgzf"], res["block_csize"], int(res["line_start"][-1]), lib.DEF_CHUNK)
                    index.add(writer, res, base)
                    filtered_count += res["n_filtered"]
                    first += res["n_records"]
                    pieces[k] = None
        except lib.UgvcDataError as err:
            if getattr(err, "afr_record", -1) >= 0:
                rec = first + err.afr_record
                if err.afr_reason == lib.AFR_E_TYPE:
                    raise TypeError(f"record {rec}: len() of a Number=1 VAF / BG_VAF "
                                    f"(object of type 'float' has no len())") from err
                raise lib.UgvcDataError(err.code, f"record {rec}: a GT / VAF / BG_VAF literal that cannot be "
                                                  f"parsed") from err
            raise
        writer.close()
        index.write(final + ".tbi")
    finally:
        ctx.close()
    logger.info(f"Filtered {filtered_count} variants with {new_filter} filter.")
    logger.info(f"Annotated VCF written to: {output_vcf}")


def run(argv: list[str]):
    "Annotate variants with low AF ratio"
    logging.basicConfig(format="%(asctime)s %(message)s", level=logging.INFO)
    args = parse_args(argv)
    filter_low_af_ratio_to_background(
        input_vcf=args.input_vcf,
        output_vcf=args.output_vcf,
        af_ratio_threshold=args.af_ratio_threshold,
        af_ratio_threshold_h_indels=args.af_ratio_threshold_h_indels,
        t_vaf_threshold=args.tumor_vaf_threshold_h_indels,
        new_filter=args.new_filter,
        device=args.device,
    )


def main():
    import sys

    run(sys.argv[1:])


if __name__ == "__main__":
    main()
