"""Seeded DeepVariant-like gVCF records for the gvcf_hcr tests (tests/test_gvcf_hcr_*.py, tests/test_gpu_gvcf_hcr.py,
scripts/make_golden_gvcf_hcr.py, scripts/bench_gvcf_hcr.py): reference blocks with END and a <*> ALT, variant records,
deletions whose REF covers the following blocks, RefCall deletions, several contigs; plus a crafted corpus of the rule's
edges and the error records."""
from __future__ import annotations

import numpy as np

CONTIGS = (("chr1", 10_000_000), ("chr2", 8_000_000), ("chr3", 6_000_000), ("chrX", 4_000_000), ("chrM", 16569))


def header(gq: str | None = "Number=1,Type=Integer", info_end: bool = True, contigs=CONTIGS) -> list[str]:
    lines = ["##fileformat=VCFv4.2", '##FILTER=<ID=PASS,Description="All filters passed">',
             '##FILTER=<ID=RefCall,Description="Genotyping model thinks this site is reference.">']
    if info_end:
        lines.append('##INFO=<ID=END,Number=1,Type=Integer,Description="End position (for use with symbolic alleles)">')
    lines.append('##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">')
    if gq is not None:
        lines.append(f'##FORMAT=<ID=GQ,{gq},Description="Conditional genotype quality">')
    lines += ['##FORMAT=<ID=DP,Number=1,Type=Integer,Description="Read depth">',
              '##FORMAT=<ID=MIN_DP,Number=1,Type=Integer,Description="Minimum DP observed within the GVCF block.">',
              '##FORMAT=<ID=PL,Number=G,Type=Integer,Description="Phred-scaled genotype likelihoods">']
    lines += [f"##contig=<ID={c},length={n}>" for c, n in contigs]
    lines.append("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tsample")
    return lines


def text(records: list[str], **kw) -> str:
    return "\n".join(header(**kw)) + "\n" + "".join(r + "\n" for r in records)


def block(chrom: str, pos: int, end: int, gq, ref: str = "A") -> str:
    return f"{chrom}\t{pos}\t.\t{ref}\t<*>\t0\t.\tEND={end}\tGT:GQ:MIN_DP:PL\t0/0:{gq}:20:0,{gq},99"


def var(chrom: str, pos: int, ref: str, alt: str, gt: str = "0/1", gq="30", flt: str = "PASS", fmt: str = "GT:GQ:DP:PL",
        sample: str | None = None) -> str:
    s = sample if sample is not None else f"{gt}:{gq}:25:30,0,40"
    return f"{chrom}\t{pos}\t.\t{ref}\t{alt},<*>\t20.5\t{flt}\t.\t{fmt}\t{s}"


def random_records(n: int, seed: int, contigs=("chr1", "chr2", "chr3"), overlap: float = 1.0) -> list[str]:
    """n records over `contigs` in order: about 70 % reference blocks (1..200 bases), SNVs, insertions, deletions of
    2..40 bases whose following blocks overlap them (skipped), RefCall deletions (GT ./. or 0/0: their first base only)
    and variants that a block overlaps by a few bases; GQ 0..99."""
    rng = np.random.default_rng(seed)
    per = np.diff(np.linspace(0, n, len(contigs) + 1).astype(int))
    out: list[str] = []
    bases = "ACGT"
    for chrom, m in zip(contigs, per):
        pos = int(rng.integers(1, 50))
        for _ in range(m):
            u = rng.random()
            gq = int(rng.integers(0, 100)) if rng.random() < 0.6 else int(rng.integers(15, 26))
            ref0 = bases[int(rng.integers(4))]
            if u < 0.70:
                ln = int(rng.geometric(0.02)) if rng.random() < 0.8 else int(rng.integers(1, 4))
                out.append(block(chrom, pos, pos + ln - 1, gq, ref0))
                pos += ln if rng.random() > 0.03 * overlap else max(1, ln - int(rng.integers(1, 4)))
            elif u < 0.82:
                out.append(var(chrom, pos, ref0, bases[(bases.index(ref0) + 1) % 4], gq=gq))
                pos += 1 if rng.random() > 0.1 * overlap else 0
            elif u < 0.87:
                out.append(var(chrom, pos, ref0, ref0 + "TT", gt="1/1", gq=gq))
                pos += 1
            elif u < 0.94:
                dl = int(rng.integers(2, 41))
                ref = "".join(bases[int(x)] for x in rng.integers(0, 4, dl))
                out.append(var(chrom, pos, ref, ref[0], gt="0/1" if rng.random() < 0.7 else "1/1", gq=gq))
                pos += 1 if rng.random() < 0.7 * overlap else dl
            else:
                dl = int(rng.integers(2, 30))
                ref = "".join(bases[int(x)] for x in rng.integers(0, 4, dl))
                gt = ("./.", "0/0", "0|0")[int(rng.integers(3))]
                out.append(var(chrom, pos, ref, ref[0], gt=gt, gq=gq, flt="RefCall"))
                pos += 1
    return out


def alternating(n: int, chrom: str = "chr1", pos0: int = 100, gq=30) -> list[str]:
    """A record at every position, each two bases long: every record overlaps the next, so after the first there is no
    reset point and the kept records are every second one."""
    return [var(chrom, pos0 + k, "AC", "A", gq=gq) for k in range(n)]


def crafted_records() -> list[tuple[str, list[str]]]:
    """(name, records) of the rule's edges, each error-free under the default header."""
    c = []
    c.append(("refcall_gts", [var("chr1", 100 + 10 * k, "ACGT", "A", gt=g, flt="RefCall")
                              for k, g in enumerate(("0/0", "0|0", "./.", ".", "0", "0/1", "1/1", "./0", "0/0/0"))]
              + [var("chr1", 300, "ACGT", "A", fmt="GT:DP:PL", sample="0/0:25:30,0,40"),
                 var("chr1", 320, "ACGT", "A", fmt="DP:GQ:GT", sample="25:40:0/1")]))
    c.append(("end_vs_pos", [block("chr1", 1000, 999, 30), block("chr1", 1001, 1001, 30), block("chr1", 1002, 1010, 30),
                             f"chr1\t1011\t.\tACG\t<*>\t0\t.\tEND=1011\tGT:GQ\t0/0:50",
                             f"chr1\t1020\t.\tA\t<*>\t0\t.\tEND=10x\tGT:GQ\t0/0:50",
                             f"chr1\t1030\t.\tA\t<*>\t0\t.\tDP=3;END=1040;END=1100\tGT:GQ\t0/0:50",
                             f"chr1\t1041\t.\tA\t<*>\t0\t.\tEND=\tGT:GQ\t0/0:50"]))
    c.append(("long_deletion", [var("chr1", 2000, "A" * 60, "A", gt="0/1", gq=40)]
              + [block("chr1", 2001 + 5 * k, 2005 + 5 * k, 30 + k) for k in range(14)]
              + [block("chr1", 2071, 2080, 30)]))
    c.append(("nested_and_chained", [block("chr1", 3000, 3100, 30), var("chr1", 3010, "ACGTACGT", "A", gq=60),
                                     block("chr1", 3050, 3150, 99), block("chr1", 3101, 3120, 10),
                                     block("chr1", 3121, 3160, 45), block("chr1", 3151, 3200, 45),
                                     block("chr1", 3161, 3170, 45)]))
    c.append(("contig_change_after_overlap", [block("chr1", 4000, 9000, 30), var("chr1", 4500, "A", "T", gq=60),
                                              block("chr2", 10, 20, 30), block("chr2", 15, 30, 30),
                                              block("chr2", 21, 40, 30), block("chr3", 1, 1, 30)]))
    c.append(("gq_on_skipped", [block("chr1", 5000, 5100, 30), block("chr1", 5050, 5060, "."),
                                var("chr1", 5070, "A", "C", fmt="GT:GQ", sample="0/1"),
                                var("chr1", 5080, "A", "C", fmt="GT:DP", sample="0/1:5")]))
    c.append(("book_ended_and_gapped", [block("chr1", 6000, 6009, 30), block("chr1", 6010, 6019, 35),
                                        block("chr1", 6020, 6029, 5), block("chr1", 6030, 6039, 30),
                                        block("chr1", 6041, 6050, 30), block("chr1", 6051, 6051, 20),
                                        block("chr1", 6052, 6060, 19), block("chr1", 6061, 6070, 99),
                                        var("chr1", 6071, "AC", "A", gt="0/0", gq=30),
                                        block("chr1", 6072, 6080, 30)]))
    c.append(("gq_absent", [var("chr1", 7000, "A", "C", fmt="GT:DP", sample="0/1:4"),
                            var("chr1", 7001, "ACG", "A", fmt="GT:DP", sample="0/1:4"), block("chr1", 7002, 7010, 0),
                            f"chr1\t7020\t.\tA\tC\t9\tPASS\t.", f"chr1\t7030\t.\tA\tC\t9\tPASS\t.\t.\t."]))
    c.append(("end_to_contig_end", [block("chr2", 100, 8_000_000, 30)] + [block("chr2", 200 + 10 * k, 205 + 10 * k, 40)
                                                                         for k in range(20)] + [block("chr3", 5, 9, 30)]))
    return c


def error_records() -> list[tuple[str, str, dict]]:
    """(record, kind, header kwargs) of a record where the tool raises when it is the only kept candidate: kind is
    "type" (TypeError), "key" (KeyError) or "literal" (a literal that cannot be typed)."""
    return [
        (block("chr1", 500, 510, "."), "type", {}),
        (var("chr1", 500, "A", "C", fmt="GT:GQ", sample="0/1"), "type", {}),
        (var("chr1", 500, "A", "C", gq="30,40"), "type", {"gq": "Number=.,Type=Integer"}),
        (var("chr1", 500, "A", "C", gq="30"), "type", {"gq": "Number=1,Type=String"}),
        (var("chr1", 500, "A", "C", gq="30"), "type", {"gq": None}),
        (var("chr1", 500, "ACG", "A", fmt="GQ:DP", sample="30:5"), "key", {}),
        (var("chr1", 500, "A", "C", gq="3x"), "literal", {}),
        (var("chr1", 500, "A", "C", gt="0/x"), "literal", {}),
    ]
