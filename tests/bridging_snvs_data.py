"""Inputs of the calibrate_bridging_snvs tests: a seeded genome (homopolymer runs, soft-masked stretches, N runs, a short
contig for the contig ends), a crafted corpus of records at the edges of every branch of the tool, records that raise,
and seeded random tumor/normal records."""
from __future__ import annotations

import numpy as np

BASES = np.frombuffer(b"ACGT", np.uint8)


def genome(seed: int = 7, lengths=(("chr1", 4000), ("chr2", 3000), ("chrM", 12))) -> dict:
    """{name: raw bytes}: runs of one base (lengths 1..9, some long), about a tenth of each contig soft-masked, N runs."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, n in lengths:
        parts, total = [], 0
        while total < n:
            run = int(rng.choice([1, 1, 1, 2, 2, 3, 4, 5, 6, 7, 8, 9]))
            parts.append(np.full(run, BASES[rng.integers(0, 4)], np.uint8))
            total += run
        seq = np.concatenate(parts)[:n].copy()
        for _ in range(max(1, n // 400)):
            a = int(rng.integers(0, n))
            seq[a: a + int(rng.integers(5, 40))] |= 0x20  # lower case
            a = int(rng.integers(0, n))
            seq[a: a + int(rng.integers(2, 12))] = ord("N")
        out[name] = seq.tobytes()
    return out


def header(n_samples: int = 2, ad: str | None = "Number=R,Type=Integer", dp: str | None = "Number=1,Type=Integer",
           bg_ad: str | None = "Number=R,Type=Integer", bg_dp: str | None = "Number=1,Type=Integer",
           contigs=("chr1", "chr2", "chrM")) -> str:
    lines = ["##fileformat=VCFv4.2", '##FILTER=<ID=RefCall,Description="Reference call">',
             '##FILTER=<ID=LowQual,Description="low">', '##INFO=<ID=END,Number=1,Type=Integer,Description="End">',
             '##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">']
    for key, decl in (("AD", ad), ("DP", dp), ("BG_AD", bg_ad), ("BG_DP", bg_dp)):
        if decl:
            lines.append(f'##FORMAT=<ID={key},{decl},Description="{key}">')
    lines += [f"##contig=<ID={c},length=100000>" for c in contigs]
    lines.append("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(f"S{k}" for k in range(n_samples)))
    return "\n".join(lines) + "\n"


def rec(chrom, pos, ref, alt, qual="8", flt="LowQual", fmt="GT:AD:DP:BG_AD:BG_DP", s0="0/1:10,8:18:20,0:20",
        s1="0/0:20,0:20:20,0:20", info=".") -> str:
    return "\t".join([chrom, str(pos), ".", ref, alt, qual, flt, info, fmt, s0, s1])


def hmer_sites(g: dict, chrom: str, min_run: int = 3) -> list[tuple[int, str, str]]:
    """(1-based pos, REF, ALT) of SNVs next to a run of at least min_run equal bases: the base just after the run made
    equal to the run's base (the bridging case)."""
    seq = g[chrom]
    out = []
    k = 0
    while k < len(seq):
        j = k
        while j < len(seq) and seq[j] == seq[k]:
            j += 1
        if j - k >= min_run and j < len(seq) and seq[j] != seq[k]:
            out.append((j + 1, chr(seq[j]), chr(seq[k])))
        k = j
    return out


def crafted_records(g: dict) -> list[str]:
    """Records at the edges of the candidate test, the window, the walks and the rescue (some raise, depending on the
    parameters)."""
    sites = hmer_sites(g, "chr1", 3)
    out = []
    for pos, ref, alt in sites[:40]:
        out.append(rec("chr1", pos, ref, alt))
        out.append(rec("chr1", pos, ref, alt, flt="."))
        out.append(rec("chr1", pos, ref, alt, flt="PASS"))
        out.append(rec("chr1", pos, ref, alt, flt="LowQual;PASS"))
        out.append(rec("chr1", pos, ref, alt, qual="5"))
        out.append(rec("chr1", pos, ref, alt, qual="4.9"))
        out.append(rec("chr1", pos, ref, alt, qual="nan"))
        out.append(rec("chr1", pos, ref, alt.lower()))
        out.append(rec("chr1", pos, ref, alt, s0="0/1:10,2:18:20,0:20"))     # tumor VAF low
        out.append(rec("chr1", pos, ref, alt, s0="0/1:10,8:18:20,3:20"))     # normal VAF high
        out.append(rec("chr1", pos, ref, alt, s0="0/1:10,8:18:20,2:20"))     # normal VAF == 0.1
        out.append(rec("chr1", pos, ref, alt, s0="0/1:10,8:18:20,0:10"))     # normal depth == 10
        out.append(rec("chr1", pos, ref, alt, s0="0/1:10,8,1:18:20,0,0:11"))
        out.append(rec("chr1", pos, ref, "*"))
        out.append(rec("chr1", pos, ref, alt + ",C"))
        out.append(rec("chr1", pos, ref + "A", alt))
        out.append(rec("chr1", pos, ref, alt + "A"))
    # soft-masked and N stretches, both contigs, the short contig and its ends
    for chrom in ("chr2", "chrM"):
        for pos, ref, alt in hmer_sites(g, chrom, 2)[:30]:
            out.append(rec(chrom, pos, ref, alt))
            out.append(rec(chrom, pos, ref, alt.lower()))
    for pos in range(1, len(g["chrM"]) + 4):
        for alt in "ACGTNa":
            out.append(rec("chrM", pos, "A", alt, s0="0/1:1,30:31:40,0:40"))
    for pos in range(1, 40):
        base = chr(g["chr1"][pos - 1]) if pos <= len(g["chr1"]) else "A"
        for alt in "ACGT":
            out.append(rec("chr1", pos, base, alt, s0="0/1:1,30:31:40,0:40"))
    # values: Float-typed depths, NaN, dropped sub-fields, empty, a 0 normal depth
    for s0 in ("0/1:10,8:18:20,0:0", "0/1:10,8:18:20,0:-3", "0/1:10,8:18:20,0", "0/1:10,8:18:20,0:", "0/1:10,8:18:.,.:20",
               "0/1:10,8:18::20", "0/1:.:18:20,0:20", "0/1:10,.:18:20,0:20", "0/1:10:18:20:20", "0/1:10,8:1:20,0:20"):
        for pos, ref, alt in sites[:6]:
            out.append(rec("chr1", pos, ref, alt, s0=s0))
    return out


def error_records(g: dict) -> list[tuple[str, str]]:
    """(record, error kind) pairs: each record raises in the reference (or is a refused literal)."""
    pos, ref, alt = hmer_sites(g, "chr1", 5)[0]
    return [
        (rec("chr1", pos, ref, "."), "type"),                                        # len(None)
        (rec("chr1", pos, ref, alt, qual="."), "type"),                              # None >= min_initial_qual
        (rec("chr1", pos, ref, alt, s0="0/1:10,8:18:20,0:."), "type"),               # max(0.01, None)
        (rec("chr1", pos, ref, alt, s0="0/1:.:18:20,0:20", fmt="GT:DP:AD:BG_AD:BG_DP"), "type"),  # 0 / None
        (rec("chr1", pos, ref, alt, s0="0/1:10,.:18:20,0:20"), "type"),              # None in sum(AD[1:])
        (rec("chr1", pos, ref, alt, s0="0/1:10,8:.:20,0:20"), "type"),               # x / None
        (rec("chr1", pos, ref, alt, s0="0/1:10,8:18:20,.:20"), "type"),              # None in sum(BG_AD[1:])
        (rec("chr1", pos, ref, alt, s0="0/1:10,8:0:20,0:20"), "zero"),               # DP == 0
        (rec("chr1", pos, ref, alt, fmt="GT:AD:DP:BG_AD"), "key"),                   # no BG_DP
        (rec("chr1", pos, ref, alt, fmt="GT:DP:BG_AD:BG_DP", s0="0/1:18:20,0:20"), "key"),
        (rec("chr1", pos, ref, alt, fmt="GT:AD:BG_AD:BG_DP", s0="0/1:10,8:20,0:20"), "key"),
        (rec("chr1", pos, ref, alt, fmt="GT:AD:DP:BG_DP", s0="0/1:10,8:18:20"), "key"),
        (rec("chr1", pos, ref, alt, fmt=".", s0="."), "key"),
        (rec("chrZ", pos, ref, alt), "fetch"),                                       # contig not in the FASTA
        (rec("chr1", 3, "A", "A"), "fetch"),                                         # pos - m - 1 < 0
        (rec("chr1", pos, ref, alt, qual="3x"), "literal"),
        (rec("chr1", pos, ref, alt, qual=""), "literal"),
        (rec("chr1", pos, ref, alt, s0="0/1:10,8:1.5:20,0:20"), "literal"),
        (rec("chr1", pos, ref, alt, s0="0/1:10,8q:18:20,0:20"), "literal"),
        (rec("chr1", 40, "A", "C", flt="PASS", s0="0/1:10,8:18:20,0:x"), "literal"),  # typed whether or not reached
    ]


def random_records(g: dict, n: int, seed: int, contigs=("chr1", "chr2")) -> list[str]:
    """Seeded random records over the contigs, sorted; about half sit on a homopolymer edge.  None of them raises with
    min_query_hmer_size <= 6."""
    rng = np.random.default_rng(seed)
    per = np.sort(rng.integers(0, len(contigs), n))
    sites = {c: [x for x in hmer_sites(g, c, 2) if x[0] >= 8] for c in contigs}
    quals = np.array(["3", "5", "4.9", "10", "20", "nan", "1e1", "0", "8", "8"])
    flts = np.array(["LowQual", ".", "PASS", "RefCall", "LowQual;RefCall", "A;PASS"])
    rows = []
    for i in range(n):
        c = contigs[per[i]]
        seq = g[c]
        if rng.random() < 0.5:
            pos, ref, alt = sites[c][int(rng.integers(0, len(sites[c])))]
        else:
            pos = int(rng.integers(8, len(seq) + 3))
            ref = chr(seq[pos - 1]) if pos <= len(seq) else "A"
            alt = "ACGTacgtN"[int(rng.integers(0, 9))]
        if rng.random() < 0.05:
            ref += "C"
        if rng.random() < 0.05:
            alt += ",T"
        dp = int(rng.integers(1, 60))
        alt_n = int(rng.integers(0, dp + 1))
        bg_dp = int(rng.integers(0, 40))
        bg_alt = int(rng.integers(0, 4))
        s0 = f"0/1:{dp - alt_n},{alt_n}:{dp}:{max(0, bg_dp - bg_alt)},{bg_alt}:{bg_dp}"
        rows.append((c, pos, rec(c, pos, ref, alt, qual=quals[rng.integers(0, quals.size)],
                                 flt=flts[rng.integers(0, flts.size)], s0=s0,
                                 info="." if rng.random() < 0.9 else f"END={pos + int(rng.integers(0, 9))}")))
    rows.sort(key=lambda r: (contigs.index(r[0]), r[1]))
    return [r[2] for r in rows]


def text(records: list[str], **hdr) -> str:
    return header(**hdr) + "".join(r + "\n" for r in records)


def params(header_text: str, **kw):
    """The BsnParams of a header and keyword arguments, from the product's header reader."""
    from variantcalling_b200 import bridging_snvs
    from variantcalling_b200.vcf_header import VcfHeader

    return bridging_snvs.bsn_params(VcfHeader(header_text), **kw)
