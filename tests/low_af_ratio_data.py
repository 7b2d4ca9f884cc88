"""Inputs of the filter_low_af_ratio_to_background tests: the reference unit test's VCF (a data fixture), a crafted corpus
of headers and records at the edges of the rule and of the FILTER edit, and seeded random multi-sample records."""
from __future__ import annotations

import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
UNIT_VCF = os.path.join(HERE, "golden", "low_af_ratio_unit.vcf")


def unit_text() -> str:
    return open(UNIT_VCF).read()


def header(n_samples: int, vaf: str = "Number=A,Type=Float", bg: str = "Number=A,Type=Float",
           vt: str | None = "Number=1,Type=String", extra: tuple[str, ...] = (), contigs=("chr1", "chr2", "chr3")) -> str:
    lines = ["##fileformat=VCFv4.2", '##FILTER=<ID=RefCall,Description="Reference call">',
             '##FILTER=<ID=LowQual,Description="low">']
    lines += list(extra)
    if vt is not None:
        lines.append(f'##INFO=<ID=VARIANT_TYPE,{vt},Description="Type of variant">')
    lines.append('##INFO=<ID=END,Number=1,Type=Integer,Description="End">')
    lines.append('##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">')
    lines.append('##FORMAT=<ID=DP,Number=1,Type=Integer,Description="Depth">')
    if vaf:
        lines.append(f'##FORMAT=<ID=VAF,{vaf},Description="VAF">')
    if bg:
        lines.append(f'##FORMAT=<ID=BG_VAF,{bg},Description="BG VAF">')
    lines += [f"##contig=<ID={c},length=100000000>" for c in contigs]
    lines.append("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(f"S{k}" for k in range(n_samples)))
    return "\n".join(lines) + "\n"


def _rec(pos: int, flt: str, info: str, fmt: str, samples: list[str], chrom: str = "chr1", ref: str = "A",
         alt: str = "T,G") -> str:
    return "\t".join([chrom, str(pos), ".", ref, alt, ".", flt, info, fmt, *samples])


# (FILTER, INFO, FORMAT, samples) of the crafted records: GT forms, dropped / missing values, zeros, -0, NaN, alleles
# out of range, later samples overriding earlier ones, RefCall / PASS / "." and new_filter at every place
CRAFTED = [
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01"]),
    ("PASS", "VARIANT_TYPE=h-indel", "GT:VAF:BG_VAF", ["0/1:0.5:0.4"]),
    ("PASS", "VARIANT_TYPE=h-indel", "GT:VAF:BG_VAF", ["0/1:0.1:0.4"]),
    (".", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0|1:0.5:0.5"]),
    ("LowQual", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["1:0.5:0.5"]),
    ("LowQual;RefCall", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("RefCall;LowAFRatioToBackground", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("LowAFRatioToBackground", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01"]),
    ("LowAFRatioToBackground", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("LowAFRatioToBackground;LowQual", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01"]),
    ("LowQual;LowAFRatioToBackground;Other", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("LowQual;Other;LowAFRatioToBackground", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01"]),
    ("LowAFRatioToBackground;LowQual;LowAFRatioToBackground;LowQual", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("PASS;LowAFRatioToBackground", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01"]),
    ("PASS;LowAFRatioToBackground", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("A;LowAFRatioToBackground;PASS;B", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01"]),
    ("A;LowAFRatioToBackground;PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("A;A;B", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("A;A;LowAFRatioToBackground", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01"]),
    ("PASS;A", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5"]),
    ("PASS", ".", "GT:VAF:BG_VAF", ["./.:0.5:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", [".:0.5:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:.:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:."]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:-0:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:-0.0"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:nan:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:NaN"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:inf:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:Infinity:inf"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/3:0.5,0.5:0.1,0.1"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/2:0.5:0.1,0.1"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/2:0.5,0.5:0.1"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["1/2:0.5,.:0.4,0.4"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["1/2:0.5,0.5:.,0.4"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["2/1:0.5,0.01:0.4,0.0001"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5", "0/1:0.5:0.01"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01", "0/1:0.5:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.5", "./.:0.5:0.01", "0/1", ".", "0/0:0.5:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.01", "0/1:0.5:0.5", "0/1:.:.", "0/1:0:0.2", "1/1:0.5:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "VAF:BG_VAF", ["0.5:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:BG_VAF", ["0/1:0.5"]),
    ("PASS", "VARIANT_TYPE=snp", ".", ["."]),
    ("PASS", "VARIANT_TYPE=snp;VARIANT_TYPE=h-indel", "GT:VAF:BG_VAF", ["0/1:0.5:0.4"]),
    ("PASS", "VARIANT_TYPE", "GT:VAF:BG_VAF", ["0/1:0.5:0.4"]),
    ("PASS", "END=2000;VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.5:0.4"]),
    ("PASS", "END=abc", "GT:VAF:BG_VAF:GT", ["0/1:0.5:0.4:1/1"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:DP:VAF:BG_VAF", ["0/1:10:0.5,0.25:0.01,0.5"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:1e-3:2E-4"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1:0.1:0.01"]),
    ("PASS", "VARIANT_TYPE=snp", "GT:VAF:BG_VAF", ["0/1::0.5"]),
]


def crafted_records(new_filter: str = "LowAFRatioToBackground") -> list[str]:
    out = []
    for k, (flt, info, fmt, samples) in enumerate(CRAFTED):
        out.append(_rec(100 + 10 * k, flt.replace("LowAFRatioToBackground", new_filter), info, fmt, samples))
    return out


def crafted_text(n_samples_pad: int = 5, **hdr) -> str:
    """The crafted records with every line padded to n_samples_pad samples (missing ones are '.')."""
    recs = []
    for r in crafted_records():
        cols = r.split("\t")
        cols += ["."] * (9 + n_samples_pad - len(cols))
        recs.append("\t".join(cols))
    return header(n_samples_pad, **hdr) + "\n".join(recs) + "\n"


def random_text(n: int, n_samples: int, seed: int, contigs=("chr1", "chr2", "chr3"), **hdr) -> str:
    """Seeded random records over several contigs (sorted), every sample drawn from the value forms of the rule."""
    rng = np.random.default_rng(seed)
    per = np.sort(rng.integers(0, len(contigs), n))
    lines = []
    vt = np.array(["snp", "h-indel", "non-h-indel"])
    flts = np.array(["PASS", ".", "LowQual", "RefCall", "LowAFRatioToBackground", "LowQual;LowAFRatioToBackground",
                     "LowAFRatioToBackground;PASS", "A;B;A"])
    gts = np.array(["0/1", "1/1", "0/2", "1/2", "./.", ".", "0|1", "1", "2/3", "0/0"])
    vals = np.array(["0.5", "0.1", "0.01", "0", ".", "0.25", "0.9", "0.333", "1e-4", "0.05"])
    pos = 0
    last = -1
    for i in range(n):
        if per[i] != last:
            pos, last = 0, per[i]
        pos += int(rng.integers(1, 50))
        n_alt = int(rng.integers(1, 4))
        samples = []
        for _s in range(n_samples):
            u = rng.random()
            if u < 0.03:
                samples.append(".")
                continue
            gt = gts[rng.integers(0, gts.size)]
            nv = n_alt if rng.random() < 0.9 else int(rng.integers(1, 4))
            v = ",".join(vals[rng.integers(0, vals.size, nv)])
            b = ",".join(vals[rng.integers(0, vals.size, nv)])
            parts = [gt, str(int(rng.integers(0, 100))), v, b]
            if rng.random() < 0.05:
                parts = parts[: int(rng.integers(1, 4))]
            samples.append(":".join(parts))
        ref = "A" * int(rng.integers(1, 4))
        info = f"VARIANT_TYPE={vt[rng.integers(0, 3)]}" + (f";END={pos + int(rng.integers(0, 30))}" if rng.random() < 0.05 else "")
        lines.append("\t".join([contigs[per[i]], str(pos), ".", ref, ",".join(["T", "G", "C"][:n_alt]), ".",
                                flts[rng.integers(0, flts.size)], info, "GT:DP:VAF:BG_VAF", *samples]))
    return header(n_samples, contigs=contigs, **hdr) + "\n".join(lines) + "\n"


def params(header_text: str, af_ratio_threshold=10, af_ratio_threshold_h_indels=0, t_vaf_threshold=0,
           new_filter="LowAFRatioToBackground"):
    """The AfrParams of a header, from the product's header reader."""
    from variantcalling_b200 import low_af_ratio
    from variantcalling_b200.vcf_header import VcfHeader

    return low_af_ratio.afr_params(VcfHeader(header_text), af_ratio_threshold, af_ratio_threshold_h_indels, t_vaf_threshold,
                                   new_filter)
