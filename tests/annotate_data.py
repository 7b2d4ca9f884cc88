"""Synthetic inputs of annotate_concordance: a seeded genome (soft-masked and N stretches, homopolymer runs, a run that
reaches a contig end) and concordance frames over it that touch every rule of the annotation (SNPs, MNPs, hmer and
non-hmer insertions and deletions, multi-allelic rows mixing them, '*' and '<DEL>' alleles, one-allele rows, lower-case
ALTs, records near both contig ends), plus a BED file of overlapping intervals."""
import numpy as np
import pandas as pd

CONTIG_SIZES = {"chr1": 3000, "chr2": 1800, "chrM": 400}
BASES = np.array(list("ACGT"))


def make_genome(seed: int = 5, sizes: dict | None = None) -> dict:
    rng = np.random.default_rng(seed)
    out = {}
    for name, size in (sizes or CONTIG_SIZES).items():
        seq = list(rng.choice(BASES, size))
        k = 0
        while k < size - 20:  # homopolymer runs of 2..14
            k += int(rng.integers(8, 40))
            run = int(rng.integers(2, 15))
            base = str(rng.choice(BASES))
            seq[k:k + run] = [base] * min(run, size - k)
            k += run
        for _ in range(max(1, size // 600)):  # soft-masked and N stretches
            a = int(rng.integers(10, size - 40))
            b = a + int(rng.integers(5, 30))
            seq[a:b] = [c.lower() for c in seq[a:b]]
            a, m = int(rng.integers(10, size - 40)), int(rng.integers(3, 12))
            seq[a:a + m] = ["N"] * m
        seq[-7:] = ["G"] * 7  # a run that reaches the contig end
        if name == "chr2":
            seq[-4:] = ["a"] * 4  # ... soft-masked
        out[name] = "".join(seq)
    return out


def fasta_text(genome: dict, width: int = 60) -> str:
    lines = []
    for name, seq in genome.items():
        lines.append(f">{name} synthetic")
        lines.extend(seq[k:k + width] for k in range(0, len(seq), width))
    return "\n".join(lines) + "\n"


def _alt_base(rng, b):
    return str(rng.choice([x for x in "ACGT" if x != b.upper()]))


def make_rows(genome: dict, n: int, seed: int) -> list:
    """n records as (chrom, pos, ref, alleles, indel), pos 1-based and at least 5 (a GC window starting before the
    contig start is empty for these sequence objects, see DESIGN.md 4b), at most len(contig)."""
    rng = np.random.default_rng(seed)
    names = list(genome)
    weights = np.array([len(genome[c]) for c in names], dtype=np.float64)
    chroms = rng.choice(len(names), n, p=weights / weights.sum())
    kinds = rng.integers(0, 14, n)
    rows = []
    for chrom_id, kind in zip(chroms, kinds):
        chrom = names[chrom_id]
        seq = genome[chrom]
        size = len(seq)
        if rng.random() < 0.08:  # near either end
            pos = int(rng.integers(5, 15)) if rng.random() < 0.5 else int(rng.integers(size - 10, size + 1))
        else:
            pos = int(rng.integers(5, size + 1))
        ref1 = seq[pos - 1].upper() if rng.random() < 0.9 else seq[pos - 1]
        nxt = seq[pos:pos + 1].upper() or "A"
        if kind <= 3:  # SNP
            alleles = (ref1, _alt_base(rng, ref1))
            ref, indel = ref1, False
        elif kind == 4:  # MNP
            k = int(rng.integers(2, 4))
            ref = seq[pos - 1:pos - 1 + k].upper() or ref1
            alleles, indel = (ref, "".join(_alt_base(rng, b) for b in ref)), False
        elif kind == 5:  # hmer insertion of the next base
            ref, indel = ref1, True
            alleles = (ref, ref + nxt * int(rng.integers(1, 4)))
        elif kind == 6:  # non-hmer insertion
            ref, indel = ref1, True
            alleles = (ref, ref + "".join(rng.choice(BASES, int(rng.integers(2, 5)))))
        elif kind == 7:  # deletion (hmer when the deleted bases are one run)
            k = int(rng.integers(1, 5))
            ref, indel = seq[pos - 1:pos + k], True
            if rng.random() < 0.7:
                ref = ref.upper()
            alleles = (ref, ref[:1]) if len(ref) > 1 else (ref, ref + "T")
        elif kind == 8:  # multi-allelic, mixing an insertion and a deletion
            ref = seq[pos - 1:pos + 1].upper()
            alleles = (ref, ref[:1], ref + nxt) if rng.random() < 0.5 else (ref, ref + nxt * 2, ref[:1])
            indel = True
        elif kind == 9:  # '*' / <DEL> alleles
            ref, indel = ref1, bool(rng.random() < 0.5)
            alleles = (ref, "*") if rng.random() < 0.5 else (ref, "<DEL>", _alt_base(rng, ref))
        elif kind == 10:  # one-allele row
            ref, indel = ref1, bool(rng.random() < 0.3)
            alleles = (ref,)
        elif kind == 11:  # lower-case ALT (SNP or insertion)
            ref = ref1
            if rng.random() < 0.5:
                alleles, indel = (ref, _alt_base(rng, ref).lower()), False
            else:
                alleles, indel = (ref, ref + nxt.lower() * 2), True
        elif kind == 12:  # multi-allelic SNP
            ref, indel = ref1, False
            alleles = (ref, *sorted({_alt_base(rng, ref) for _ in range(3)}))
        else:  # insertion whose first non-REF allele is not the longest
            ref, indel = ref1, True
            alleles = (ref, _alt_base(rng, ref), ref + nxt * 2)
        rows.append((chrom, pos, ref, tuple(alleles), bool(indel)))
    return rows


def make_frame(genome: dict, n: int, seed: int, *, with_filter: bool = True) -> pd.DataFrame:
    rows = make_rows(genome, n, seed)
    rng = np.random.default_rng(seed + 1)
    df = pd.DataFrame({
        "chrom": pd.Series([r[0] for r in rows], dtype=object),
        "pos": np.array([r[1] for r in rows], dtype=np.int64),
        "ref": pd.Series([r[2] for r in rows], dtype=object),
        "alleles": pd.Series([r[3] for r in rows], dtype=object),
        "indel": np.array([r[4] for r in rows], dtype=bool),
        "qual": np.round(rng.random(n) * 50, 2),
    })
    if with_filter:
        choice = rng.integers(0, 4, n)
        df["filter"] = pd.Series([np.nan if c == 0 else "" if c == 1 else "PASS" if c == 2 else "LowQual;SOR"
                                  for c in choice], dtype=object)
    return df


def bed_text(genome: dict, seed: int = 3) -> str:
    """Intervals over the first two contigs only, some overlapping, with starts out of order in the file."""
    rng = np.random.default_rng(seed)
    lines = []
    for chrom in list(genome)[:2]:
        size = len(genome[chrom])
        for _ in range(12):
            a = int(rng.integers(0, size - 50))
            lines.append((chrom, a, a + int(rng.integers(5, 300))))
    rng.shuffle(lines)
    return "".join(f"{c}\t{a}\t{b}\n" for c, a, b in lines)


# (name, flow order, interval files used, filter column present)
CASES = [
    ("tgca", "TGCA", True, True),
    ("no_flow", None, False, True),
    ("acgt", "ACGT", False, True),
    ("missing_base", "TGC", True, True),
    ("no_filter", "TGCA", False, False),
]
