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
import logging
import os
import struct
import threading
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from variantcalling_b200 import bgzf_io, lib
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


def _blocks(raw: np.ndarray) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Compressed offset, compressed size and uncompressed size of every BGZF block of a file's bytes."""
    mv = memoryview(raw)
    coff, csz, usz = [], [], []
    at, n = 0, raw.size
    while at < n:
        if n - at < 28 or mv[at] != 0x1F or mv[at + 1] != 0x8B:
            raise OSError(f"not a BGZF block at byte {at}")
        xlen = struct.unpack_from("<H", mv, at + 10)[0]
        bsize, x = None, at + 12
        while x < at + 12 + xlen:
            si1, si2, slen = struct.unpack_from("<BBH", mv, x)
            if (si1, si2, slen) == (66, 67, 2):
                bsize = struct.unpack_from("<H", mv, x + 4)[0] + 1
            x += 4 + slen
        if bsize is None or at + bsize > n:
            raise OSError(f"bad BGZF block at byte {at}")
        coff.append(at)
        csz.append(bsize)
        usz.append(struct.unpack_from("<I", mv, at + bsize - 4)[0])
        at += bsize
    return np.array(coff, np.int64), np.array(csz, np.int64), np.array(usz, np.int64)


def _inflate_block(raw: np.ndarray, coff: int, csize: int) -> bytes:
    xlen = struct.unpack_from("<H", memoryview(raw), coff + 10)[0]
    return zlib.decompress(bytes(raw[coff + 12 + xlen: coff + csize - 8]), -15)


def _bgzf_cuts(path: str, raw: np.ndarray, coff, csz, ustart, data_begin: int, total: int) -> list[int]:
    """Uncompressed offsets where pieces begin (line starts), about PIECE_BYTES apart: from the .tbi linear index when
    there is one, else at the first line start of a block (that block inflated on the host)."""
    cuts = [data_begin]
    cands: list[int] = []
    if os.path.exists(path + ".tbi"):
        try:
            _, lin = bgzf_io.read_tbi(path + ".tbi", linear=True)
            voffs = np.unique(np.concatenate([v for v in lin.values()] or [np.zeros(0, np.uint64)]))
            blk = np.searchsorted(coff, (voffs >> np.uint64(16)).astype(np.int64))
            ok = (blk < coff.size) & (coff[np.minimum(blk, coff.size - 1)] == (voffs >> np.uint64(16)).astype(np.int64))
            cands = sorted(int(ustart[b] + (v & np.uint64(0xFFFF))) for b, v in zip(blk[ok], voffs[ok]))
        except OSError:
            cands = []
    if cands:
        for u in cands:
            if u - cuts[-1] >= PIECE_BYTES and u < total:
                cuts.append(u)
    else:
        b = int(np.searchsorted(ustart, cuts[-1] + PIECE_BYTES))
        while b < coff.size and ustart[b] < total:
            nl = _inflate_block(raw, int(coff[b]), int(csz[b])).find(b"\n")
            if nl >= 0 and ustart[b] + nl + 1 < total:
                cuts.append(int(ustart[b]) + nl + 1)
                b = int(np.searchsorted(ustart, cuts[-1] + PIECE_BYTES))
            else:  # a line longer than the block: the next block
                b += 1
    return cuts + [total]


def _text_cuts(text: np.ndarray, data_begin: int) -> list[int]:
    cuts = [data_begin]
    while text.size - cuts[-1] > PIECE_BYTES:
        nl = np.flatnonzero(text[cuts[-1] + PIECE_BYTES:] == 10)  # noqa: PLR2004
        if not nl.size or cuts[-1] + PIECE_BYTES + int(nl[0]) + 1 >= text.size:
            break
        cuts.append(cuts[-1] + PIECE_BYTES + int(nl[0]) + 1)
    return [*cuts, text.size]


class _Index:
    """Contig runs and tabix intervals of the written records (htslib's rules: DESIGN.md 4)."""

    def __init__(self, info_end: bool):
        self.info_end = info_end
        self.names: list[str] = []
        self.cur: list[tuple] = []
        self.sections: list[bytes] = []
        self.last_pos = -1

    def add(self, writer: bgzf_io.BgzfWriter, res: dict, base: int):
        n = res["n_records"]
        if n == 0:
            return
        ri, ls = res["recinfo"], res["line_start"]
        beg = ri["pos"].astype(np.int64) - 1
        end = beg + np.maximum(1, (ri["flags"] >> 8).astype(np.int64))
        if self.info_end:
            end = np.where(res["end"] > beg, res["end"], end)
        vs = writer.virtual_offsets(base + ls[:-1])
        ve = writer.virtual_offsets(base + ls[1:] - 1) + np.uint64(1)
        starts = np.flatnonzero(res["flags"] & lib.AFR_NEW_CONTIG)
        bounds = [*starts.tolist(), n]
        for k, r0 in enumerate(starts.tolist()):
            r1 = bounds[k + 1]
            name = self._name(res, r0)
            if not self.names or self.names[-1] != name:
                if name in self.names:
                    raise ValueError(f"records of contig {name} are not contiguous: the output cannot be indexed")
                self._close()
                self.names.append(name)
                self.last_pos = -1
            b = beg[r0:r1]
            if b[0] < self.last_pos or np.any(b[1:] < b[:-1]):
                raise ValueError(f"records of contig {name} are not sorted by position: the output cannot be indexed")
            self.last_pos = int(b[-1])
            self.cur.append((b, end[r0:r1], vs[r0:r1], ve[r0:r1]))

    @staticmethod
    def _name(res: dict, r: int) -> str:
        """CHROM of record r, read back from the call's output blocks (contig runs are few)."""
        off = int(res["line_start"][r])
        cs = res["block_csize"].astype(np.int64)
        cstart = np.concatenate(([0], np.cumsum(cs)))
        k = off // lib.DEF_CHUNK
        buf = b""
        while k < cs.size:
            buf += _inflate_block(res["bgzf"], int(cstart[k]), int(cs[k]))
            tab = buf.find(b"\t", off - (off // lib.DEF_CHUNK) * lib.DEF_CHUNK)
            if tab >= 0:
                return buf[off - (off // lib.DEF_CHUNK) * lib.DEF_CHUNK: tab].decode()
            k += 1
        raise ValueError(f"record {r} has a single column")

    def _close(self):
        if self.names:
            cols = [np.concatenate([c[k] for c in self.cur]) for k in range(4)] if self.cur else [np.zeros(0, np.int64)] * 4
            self.sections.append(bgzf_io.tbi_section(cols[0], cols[1], cols[2].astype(np.uint64), cols[3].astype(np.uint64)))
        self.cur = []

    def write(self, path: str):
        self._close()
        bgzf_io.write_tbi(path, bgzf_io.tbi_assemble(self.names, self.sections))


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
    raw = np.fromfile(input_vcf, dtype=np.uint8)
    is_bgzf = raw.size >= 2 and raw[0] == 0x1F and raw[1] == 0x8B  # noqa: PLR2004
    header_text = bgzf_io.read_header_text(input_vcf)
    header = VcfHeader(header_text)
    params = afr_params(header, af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold, new_filter)
    desc = filter_description(af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold)
    lines = output_lines(header, new_filter, desc)
    final = output_vcf if output_vcf.endswith(".gz") else output_vcf + ".gz"  # pysam.tabix_index compresses a plain file

    data_begin = len(header_text.encode())
    if is_bgzf:
        coff, csz, usz = _blocks(raw)
        ustart = np.concatenate(([0], np.cumsum(usz)))
        total = int(ustart[-1])
        cuts = _bgzf_cuts(input_vcf, raw, coff, csz, ustart[:-1], data_begin, total)
    else:
        total = raw.size
        cuts = _text_cuts(raw, data_begin)
    pieces = []
    for u0, u1 in zip(cuts[:-1], cuts[1:]):
        if u1 <= u0:
            continue
        if is_bgzf:
            b0 = int(np.searchsorted(ustart, u0, side="right")) - 1
            b1 = int(np.searchsorted(ustart, u1 - 1, side="right")) - 1
            span = int(ustart[b1 + 1] - ustart[b0])
            pieces.append((raw[coff[b0]: coff[b1] + csz[b1]], u0 - int(ustart[b0]), u1 - u0, span))
        else:
            pieces.append((raw[u0:u1], 0, u1 - u0, u1 - u0))
    if pieces and not is_bgzf and raw[cuts[-1] - 1] != 10:  # noqa: PLR2004
        raise ValueError(f"{input_vcf}: the last line has no newline")

    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    ctx = lib.Context(device)
    ctx.load_plan(MC.compile_plan_no_model(header).blob)
    cap = max([p[3] for p in pieces], default=1) + 64
    n_lanes = 2 if len(pieces) > 1 else 1
    ctx.reserve(cap, cap // 8 + 16, n_lanes)

    logger.info(f"Processing {input_vcf} and writing to {output_vcf}")
    locks = [threading.Lock() for _ in range(n_lanes)]

    def one(k: int):
        data, skip, take, _span = pieces[k]
        with locks[k % n_lanes]:
            return ctx.afr_bgzf(data, skip, take, not is_bgzf, params, cap // 8 + 16, lane=k % n_lanes)

    writer = bgzf_io.BgzfWriter(final)
    writer.write(("\n".join(lines) + "\n").encode())
    index = _Index("END" in header.info)
    filtered_count = 0
    first = 0
    try:
        with ThreadPoolExecutor(max_workers=n_lanes, thread_name_prefix="ugvc-afr") as pool:
            futures = [pool.submit(one, k) for k in range(len(pieces))]
            for k, fut in enumerate(futures):
                try:
                    res = fut.result()
                except lib.UgvcDataError as err:
                    if getattr(err, "afr_record", -1) >= 0:
                        rec = first + err.afr_record
                        if err.afr_reason == lib.AFR_E_TYPE:
                            raise TypeError(f"record {rec}: len() of a Number=1 VAF / BG_VAF "
                                            f"(object of type 'float' has no len())") from err
                        raise lib.UgvcDataError(err.code, f"record {rec}: a GT / VAF / BG_VAF literal that cannot be "
                                                          f"parsed") from err
                    raise
                base = writer.uoffset
                writer.write_compressed(res["bgzf"], res["block_csize"], int(res["line_start"][-1]), lib.DEF_CHUNK)
                index.add(writer, res, base)
                filtered_count += res["n_filtered"]
                first += res["n_records"]
                pieces[k] = None
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
