"""Host side of ``--treat_multiallelics`` (filter_variants_pipeline.py:145-166).

The reference removes every multi-allelic record and every spanning-deletion cluster from the
contig's data frame, appends 1-2 biallelic rows per removed record (REF vs strongest ALT,
strongest ALT vs second ALT; ``multiallelics.py:65-177``, ``spandel.py:11-128``), scores the
new frame and folds the two score triplets of a record back into one genotype-likelihood vector
(``variant_filtering_utils.py:346-408``).

Here the same is done on VCF *text*, so that the split rows go through the very same GPU kernels
as ordinary records:

  index pass (K0+K1, no model)  ->  recinfo / line starts of the contig
  find_overlaps()               ->  multi-allelic records and deletion clusters (vectorised
                                    equivalent of ``select_overlapping_variants``, :13-62)
  SplitPlan.build()             ->  rewritten biallelic VCF lines for the split rows (REF/ALT,
                                    QUAL, per-allele INFO/FORMAT values, X_IC/X_IL/X_HIL/X_HIN,
                                    VARIANT_TYPE, QD, GT/GQ/PL: ``extract_allele_subset_*`` +
                                    ``cleanup_multiallelics`` :503-559) appended to the untouched lines
  scored pass (K0..K3)          ->  fp64 class likelihoods of every row of that text
  SplitPlan.merge()             ->  N x W likelihood matrix in input record order

``DeviceSplitPlan`` runs find_overlaps / build / merge as CUDA kernels (csrc/multiallelic.cu, C ABI ``ugvc_ma_*``) and is
what the tool uses -- on the device file path (``DeviceSplitPlan.filter_bgzf``) chained with the inflate, both passes,
the score math, the record writer and the deflate on device pointers; ``SplitPlan`` is the same algorithm in Python -- the model the kernels were written from, kept for
differential tests and as ``UGVC_MA_HOST=1`` (A/B), like ``UGVC_K1_LEGACY`` for the generic parser.
The reference's error behaviour is kept (see DESIGN.md section 4): no multi-allelic site on a
contig -> ValueError, no deletion cluster -> KeyError('spanning_deletion'), a called genotype
without the selected alleles -> AssertionError, per-genotype (Number=G) tags other than PL ->
RuntimeError, a 2-class model -> IndexError.
"""
from __future__ import annotations

import ctypes as C
import os
import re
import struct
from dataclasses import dataclass, field

import numpy as np

STAR = "*"
FLOW_ORDER = "TGCA"
_NOT_ACGT = re.compile(r"[^ACGT]")
_NOT_REF_CHARS = re.compile(r"[^.ATCG]")


# ------------------------------------------------------------------ FASTA
def read_fasta_contig(path: str, contig: str, *, as_bytes: bool = False):
    """Sequence of one contig (via ``path.fai`` when present, else a linear scan): a ``str``, or with ``as_bytes``
    the raw bytes (what the device plan uploads; no decode / encode round trip of a 250 MB chromosome)."""
    fai = path + ".fai"
    if os.path.exists(fai):
        with open(fai) as fh:
            for ln in fh:
                name, length, offset, bases, width = ln.rstrip("\n").split("\t")[:5]
                if name == contig:
                    length, offset, bases, width = int(length), int(offset), int(bases), int(width)
                    n_lines = (length + bases - 1) // bases
                    with open(path, "rb") as fa:
                        fa.seek(offset)
                        raw = fa.read(length + n_lines * (width - bases))
                    seq = raw.replace(b"\n", b"").replace(b"\r", b"")[:length]
                    return seq if as_bytes else seq.decode()
        raise KeyError(contig)
    seq, on = [], False
    with open(path, "rb") as fa:
        for ln in fa:
            if ln.startswith(b">"):
                if on:
                    break
                on = ln[1:].split()[0].decode() == contig if ln[1:].split() else False
            elif on:
                seq.append(ln.strip())
    if not on and not seq:
        raise KeyError(contig)
    out = b"".join(seq)
    return out if as_bytes else out.decode()


# ------------------------------------------------------------------ genotype / PL index arithmetic
def get_pl_idx(tup) -> int:
    """Triangular index of genotype (a, b) (multiallelics.py:239-252)."""
    hi, lo = max(tup), min(tup)
    return hi * (hi + 1) // 2 + lo


def select_pl_for_allele_subset(pl, pair, *, normed: bool = True) -> tuple:
    """multiallelics.py:280-308"""
    a, b = pair
    take = [pl[get_pl_idx((a, a))], pl[get_pl_idx((a, b))], pl[get_pl_idx((b, b))]]
    if normed:
        m = min(take)
        take = [v - m for v in take]
    return tuple(take)


def encode_gt_for_allele_subset(gt, pair) -> tuple:
    """multiallelics.py:206-236"""
    has0, has1 = pair[0] in gt, pair[1] in gt
    assert has0 or has1, "One of the alleles should be present in the GT"  # noqa: S101
    return (0, 1) if has0 and has1 else ((0, 0) if has0 else (1, 1))


# ------------------------------------------------------------------ flow-space hmer test
def _flow_key(seq: str) -> list:
    """Homopolymer run lengths of ``seq`` in TGCA flow order (flow_based_read.py:55-112)."""
    seq = seq.upper()
    if _NOT_ACGT.search(seq):
        raise ValueError("Input contains non ACGTacgt characters" + (f":\n{seq}" if len(seq) <= 100 else ""))  # noqa: PLR2004
    key, at, flow, n = [], 0, 0, len(seq)
    while at < n:
        base = FLOW_ORDER[flow & 3]
        end = at
        while end < n and seq[end] == base:
            end += 1
        key.append(end - at)
        at, flow = end, flow + 1
    return key


def _place(window: str, rel: int, ref_allele: str, candidates) -> list:
    """Window with each candidate allele substituted at index ``rel`` (Python slice semantics of
    apply_variants_to_reference, flow_based_concordance.py:263-339); symbolic / '*' alleles drop out."""
    left, right = window[0:rel], window[rel:len(window)][len(ref_allele):]
    return [left + a + right for a in candidates if not a.startswith("<") and STAR not in a]


def classify_hmer_indel_relative(alleles, pair, ref: str, pos: int, spandel=None) -> tuple:
    """('T'|'G'|'C'|'A', length) when the two haplotypes differ in exactly one flow, else ('.', 0)
    (multiallelics.py:385-465).  ``spandel``: (alleles, pos) of the deletion record spanning this one."""
    lo, hi = max(0, pos - 20), min(pos + 20, len(ref))
    window = _NOT_REF_CHARS.sub("A", ref[lo - 1:hi - 1].upper())
    star = STAR in (alleles[pair[0]], alleles[pair[1]])
    if star:
        if spandel is None:
            raise RuntimeError("when the alleles contain spanning deletion, the line containing the variant "
                               "that is a deletion is required")
        haps = _place(window, 20, alleles[0], [alleles[a] for a in sorted(pair) if alleles[a] != STAR])
        d_alleles, d_pos = spandel
        haps += _place(window, d_pos - (pos - 20), d_alleles[0], list(d_alleles[0:2]))[1:2]
    else:
        haps = _place(window, 20, alleles[0], [alleles[a] for a in sorted(pair)])
    if len(haps) < 2:  # noqa: PLR2004
        return (".", 0)
    k0, k1 = _flow_key(haps[0]), _flow_key(haps[1])
    if len(k0) != len(k1):
        return (".", 0)
    diff = [i for i in range(len(k0)) if k0[i] != k1[i]]
    if len(diff) != 1:
        return (".", 0)
    return (FLOW_ORDER[diff[0] % 4], max(k0[diff[0]], k1[diff[0]]))


# ------------------------------------------------------------------ overlap detection
def find_overlaps(pos: np.ndarray, n_alleles: np.ndarray, del_len: np.ndarray, has_star: np.ndarray):
    """-> (multi-allelic singles, deletion clusters), both ascending.

    Equivalent of ``select_overlapping_variants`` (multiallelics.py:13-62) without the row loop.
    From the first deletion on, the reference's loop always holds an open cluster: a row whose
    position lies beyond the running ``span = max(pos + del_len)`` of the rows before it closes the
    cluster and becomes the head of the next; any other row joins the open cluster iff it carries
    the '*' allele.  Clusters of one row are dropped, and so is the cluster still open at the end
    of the contig (the reference never flushes it).  Multi-allelic rows outside flushed clusters are
    handled one by one."""
    n = pos.size
    multi = n_alleles > 2  # noqa: PLR2004
    clusters: list[list[int]] = []
    dels = np.flatnonzero(del_len > 0)
    if dels.size:
        first = int(dels[0])
        reach = np.maximum.accumulate((pos + del_len)[first:])
        boundary = np.ones(n - first, dtype=bool)
        boundary[1:] = pos[first + 1:] > reach[:-1]
        heads = np.flatnonzero(boundary) + first
        members = np.flatnonzero(has_star[first:] & ~boundary) + first
        if members.size:
            owner = heads[np.searchsorted(heads, members, side="right") - 1]
            open_head = heads[-1]
            for h in np.unique(owner):
                if h == open_head:
                    continue
                clusters.append([int(h)] + [int(m) for m in members[owner == h]])
    in_cluster = np.zeros(n, dtype=bool)
    for c in clusters:
        in_cluster[c] = True
    singles = [int(i) for i in np.flatnonzero(multi & ~in_cluster)]
    return singles, clusters


# ------------------------------------------------------------------ record rewriting
class _Record:
    """The columns of one VCF line with the few typed views the split needs."""

    def __init__(self, line: bytes):
        self.cols = line.decode().rstrip("\n").split("\t")
        c = self.cols
        self.pos = int(c[1])
        self.alleles = (c[3],) + (() if c[4] == "." else tuple(c[4].split(",")))
        self.info = [] if c[7] == "." else [kv.partition("=") for kv in c[7].split(";") if kv]
        self.fmt = c[8].split(":") if len(c) > 9 and c[8] != "." else []  # noqa: PLR2004
        vals = c[9].split(":") if self.fmt else []
        self.sample = vals + [None] * (len(self.fmt) - len(vals))

    def info_value(self, tag):
        for k, _sep, v in self.info:
            if k == tag:
                return v
        return None

    def sample_value(self, tag):
        return self.sample[self.fmt.index(tag)] if tag in self.fmt else None

    def int_tuple(self, text):
        return None if text is None else tuple(None if t in (".", "") else int(t) for t in text.split(","))

    @property
    def gt(self):
        text = self.sample_value("GT")
        if text is None:
            return (None,)
        return tuple(None if t in (".", "") else int(t) for t in re.split(r"[/|]", text))

    @property
    def pl(self):
        return self.int_tuple(self.sample_value("PL"))

    @property
    def dp(self):
        """FORMAT DP wins over INFO DP whenever the FORMAT key is there (vcftools.py:69-89)."""
        text = self.sample_value("DP") if "DP" in self.fmt else self.info_value("DP")
        return None if text in (None, ".", "") else int(text)


def _subsample(elems: list, number, pair) -> list:
    """vcftools.py:745-778 on the comma-split text of a value."""
    if number == "A":
        return [elems[i - 1] for i in pair[1:]]
    if number == "R":
        return [elems[i] for i in pair]
    if number == "G":
        raise RuntimeError("Special treatment is required for 'G' fields, not supported by this function")
    if number == ".":
        return elems
    raise RuntimeError(f"Number {number} is not supported")


def _float_text(v: float) -> str:
    if v != v:  # noqa: PLR0124  (NaN -> missing: same imputation downstream)
        return "."
    if v in (float("inf"), float("-inf")):
        return "inf" if v > 0 else "-inf"
    return repr(float(v))


@dataclass
class _Group:
    origin: int                 # record index in the contig
    rows: list = field(default_factory=list)       # indices into SplitPlan.split_lines
    second_alleles: tuple | None = None            # alleles of the (strongest, second) row
    n_alleles: int = 2
    orig_alleles: tuple = ()


class SplitPlan:
    """Built per contig from the index pass; owns the text of the scored pass and the merge."""

    SPECIAL = ("sb", "pl", "gt", "ref", "indel", "x_ic", "x_il", "x_hil", "x_hin", "label")

    def __init__(self, header, loaded_columns: dict, ref_seq: str):
        self.header = header
        self.ref = ref_seq
        # column (lower-cased tag) -> Number, FORMAT winning over INFO, with the reference's overrides
        # (header_record_number, vcftools.py:687-742)
        num = {}
        for table in (header.info, header.formats):
            for tag, (number, _t) in table.items():
                num[tag.lower()] = int(number) if number.isdigit() else number
        for k in ("hapcomp", "hapdom"):
            if num.get(k) == "A":
                num[k] = 1
        num.update({"rpa": "R", "ru": 1, "str": 1})
        self.numbers = num
        # per source table: column -> how to sub-sample its values (None: leave the text alone)
        self.rule = {}
        for is_format, table in ((False, header.info), (True, header.formats)):
            for tag, (number, _t) in table.items():
                col = tag.lower()
                multi_valued = number not in ("0", "1") and num[col] != 1
                self.rule.setdefault((is_format, col), num[col] if multi_valued else None)
        self.loaded = set(loaded_columns)          # lower-cased columns the loader keeps
        self.loaded_tags = set(loaded_columns.values())
        self.split_lines: list[bytes] = []
        self.groups: list[_Group] = []
        self.kept: np.ndarray | None = None

    # ---- one biallelic row over `pair`
    def _rewrite(self, rec: _Record, pair, spandel: _Record | None) -> dict:
        """-> dict(cols, x_il, x_hil, pl, dp, vt) of the new row before clean-up."""
        alleles = rec.alleles
        a0, a1 = alleles[pair[0]], alleles[pair[1]]
        star = STAR in (a0, a1)
        if star and spandel is None:
            raise RuntimeError("Can't deal with spanning deletion allele without the spandel")
        indel = True if star else (len(a0) != len(a1))
        if not indel:
            x_ic, x_il = "NA", None
        elif star:
            il = rec.int_tuple(spandel.info_value("X_IL"))
            x_ic, x_il = "del", il[0]
        elif len(a0) > len(a1):
            x_ic, x_il = "del", len(a0) - len(a1)
        else:
            x_ic, x_il = "ins", len(a1) - len(a0)
        hin, hil = classify_hmer_indel_relative(alleles, pair, self.ref, rec.pos,
                                                None if spandel is None else (spandel.alleles, spandel.pos))
        special_info = {"x_ic": x_ic, "x_il": "." if x_il is None else str(x_il), "x_hil": str(hil), "x_hin": hin}
        in_format = {k.lower() for k in rec.fmt}

        def convert(col, text, is_format):
            """Per-allele values of a loaded, multi-valued tag -> the pair's values."""
            if col not in self.loaded or col in self.SPECIAL or text is None:
                return text
            if not is_format and col in in_format:
                return text  # the FORMAT value is the one the loader keeps
            number = self.rule.get((is_format, col))
            if number is None:
                return text
            return ",".join(_subsample(text.split(","), number, pair))

        info, seen = [], set()
        for k, sep, v in rec.info:
            col = k.lower()
            if col in special_info and col in self.loaded:
                info.append(f"{k}={special_info[col]}")
                seen.add(col)
            elif sep:
                info.append(f"{k}={convert(col, v, False)}")
            else:
                info.append(k)
        for col, val in special_info.items():
            if col in self.loaded and col not in seen:
                info.append(f"{self.header_tag(col)}={val}")
        pl = select_pl_for_allele_subset(rec.pl, pair)
        fmt, sample = list(rec.fmt), []
        for k, v in zip(rec.fmt, rec.sample):
            col = k.lower()
            if k == "GT":
                sample.append("/".join(str(g) for g in encode_gt_for_allele_subset(rec.gt, pair)))
            elif k == "PL":
                sample.append(",".join(str(x) for x in pl))
            else:
                sample.append(convert(col, "." if v is None else v, True))
        # '*' cannot be told from a base by its length: write it one longer than REF so that the
        # loader-derived `indel` is True, as the reference sets it for spanning deletions
        alt = a1 if a1 != STAR else STAR * (len(a0) + 1)
        cols = rec.cols[:3] + [a0, alt] + rec.cols[5:7] + [info, fmt, sample] + rec.cols[10:]
        return {"cols": cols, "x_il": x_il, "x_hil": hil, "pl": pl, "dp": rec.dp,
                "vt": rec.info_value("VARIANT_TYPE"), "alleles": (a0, a1)}

    def header_tag(self, col: str) -> str:
        for table in (self.header.info, self.header.formats):
            for t in table:
                if t.lower() == col:
                    return t
        return col.upper()

    @staticmethod
    def _as_is(rec: _Record) -> dict:
        il = rec.int_tuple(rec.info_value("X_IL"))
        hil = rec.int_tuple(rec.info_value("X_HIL"))
        info = [f"{k}={v}" if sep else k for k, sep, v in rec.info]
        return {"cols": rec.cols[:7] + [info, list(rec.fmt), ["." if v is None else v for v in rec.sample]] + rec.cols[10:],
                "x_il": il[0], "x_hil": hil[0], "pl": rec.pl, "dp": rec.dp, "vt": rec.info_value("VARIANT_TYPE"),
                "alleles": rec.alleles}

    # ---- cleanup_multiallelics (multiallelics.py:503-559) on one row, then serialise
    def _finish(self, row: dict) -> bytes:
        vt, il, hil, pl = row["vt"], row["x_il"], row["x_hil"], row["pl"]
        if vt == "snp" and il is not None and il != 0:
            vt = "non-h-indel"
        if vt == "non-h-indel" and hil is not None and hil > 0:
            vt = "h-indel"
        if vt == "h-indel" and (hil is None or hil == 0):
            vt = "non-h-indel"
        ordered = sorted(pl)
        gq = min(99, max(0, ordered[1] - ordered[0]))
        qual = max(0, min(pl[1:]) - pl[0])
        dp = row["dp"]
        if dp is None:
            qd = float("nan")
        elif dp == 0:
            qd = float("nan") if qual == 0 else float("inf")
        else:
            qd = qual / dp
        cols = row["cols"]
        info, fmt, sample = cols[7], cols[8], cols[9]

        def put_info(tag, text, *, add):
            for i, kv in enumerate(info):
                if kv.split("=", 1)[0] == tag:
                    info[i] = f"{tag}={text}"
                    return
            if add:
                info.append(f"{tag}={text}")

        if vt is not None:
            put_info("VARIANT_TYPE", vt, add=False)
        if "QD" in self.header.info:
            put_info("QD", _float_text(qd), add=True)
        if "GQ" in self.header.formats:
            if "GQ" in fmt:
                sample[fmt.index("GQ")] = str(gq)
            else:
                fmt.append("GQ")
                sample.append(str(gq))
        out = cols[:5] + [str(qual), cols[6], ";".join(info) if info else ".", ":".join(fmt), ":".join(sample)] + cols[10:]
        return "\t".join(out).encode() + b"\n"

    # ---- groups
    def _split_plain(self, rec: _Record) -> list:
        """split_multiallelic_variants (multiallelics.py:65-127): allele pairs to genotype."""
        n = len(rec.alleles)
        hom = np.array([select_pl_for_allele_subset(rec.pl, (0, i), normed=False)[-1] for i in range(1, n)])
        absent = np.array([i not in rec.gt for i in range(1, n)])
        order = [int(x) for x in np.argsort(hom + absent * 1000, kind="stable") + 1 if rec.alleles[x] != STAR]
        return [(0, order[0])] if len(order) == 1 else [(0, order[0]), (order[0], order[1])]

    @staticmethod
    def _split_spanned(rec: _Record) -> list:
        """split_multiallelic_variants_with_spandel (spandel.py:11-63): '*' is forced to be weakest."""
        n = len(rec.alleles)
        star = rec.alleles.index(STAR)
        keys = [select_pl_for_allele_subset(rec.pl, (0, i), normed=False)[-1] + 100000 * (i == star) for i in range(1, n)]
        order = [int(x) for x in np.argsort(np.array(keys), kind="stable") + 1]
        return [(0, order[0]), (order[0], order[1])]

    def _add_group(self, origin: int, rec: _Record, rows: list):
        g = _Group(origin=origin, n_alleles=len(rec.alleles), orig_alleles=rec.alleles)
        for row in rows:
            g.rows.append(len(self.split_lines))
            self.split_lines.append(self._finish(row))
        if len(rows) == 2:  # noqa: PLR2004
            g.second_alleles = rows[1]["alleles"]
        self.groups.append(g)

    def build(self, text: np.ndarray, line_start: np.ndarray, recinfo: np.ndarray) -> np.ndarray:
        """-> the text of the scored pass: untouched lines in input order, then the split rows
        (multi-allelic groups, then deletion clusters), the row order of the reference's frame
        (training_prep.py:284-286)."""
        n = recinfo.size
        flags = recinfo["flags"].astype(np.int64)
        pos = recinfo["pos"].astype(np.int64)
        n_alleles = (flags >> 1) & 0x7F
        ref_len = flags >> 8
        view = memoryview(text)
        cache: dict[int, _Record] = {}

        def rec(i: int) -> _Record:
            r = cache.get(i)
            if r is None:
                r = cache[i] = _Record(bytes(view[int(line_start[i]):int(line_start[i + 1])]))
            return r

        def alleles_of(i: int) -> tuple:
            c = bytes(view[int(line_start[i]):int(line_start[i + 1])]).split(b"\t", 5)
            return (c[3],) + (() if c[4] == b"." else tuple(c[4].split(b",")))

        del_len = np.zeros(n, dtype=np.int64)
        for i in np.flatnonzero(ref_len > 1):  # only a REF longer than one base can be a deletion
            a = alleles_of(int(i))
            del_len[i] = max(len(a[0]) - len(y) for y in a)
        has_star = np.zeros(n, dtype=bool)
        stars = np.flatnonzero(text == 42)  # noqa: PLR2004  ('*' anywhere on the line: confirm on the ALT column)
        if stars.size:
            for i in np.unique(np.searchsorted(line_start, stars, side="right") - 1):
                if 0 <= i < n:
                    has_star[i] = b"*" in alleles_of(int(i))
        singles, clusters = find_overlaps(pos, n_alleles, del_len, has_star)

        if not singles:
            raise ValueError("No objects to concatenate")  # pd.concat([]) in training_prep.py:261
        for m in singles:
            r = rec(m)
            self._add_group(m, r, [self._rewrite(r, p, None) for p in self._split_plain(r)])
        if not clusters:
            raise KeyError("spanning_deletion")  # variant_filtering_utils.py:339 on a frame without the column
        for c in clusters:
            head = rec(c[0])
            if len(head.alleles) == 2:  # noqa: PLR2004
                self._add_group(c[0], head, [self._as_is(head)])
            else:
                self._add_group(c[0], head, [self._rewrite(head, p, None) for p in self._split_plain(head)])
            for i in c[1:]:
                r = rec(i)
                self._add_group(i, r, [self._rewrite(r, p, head) for p in self._split_spanned(r)])

        kept = np.ones(n, dtype=bool)
        kept[[g.origin for g in self.groups]] = False
        self.kept = kept
        pieces = []
        edges = np.flatnonzero(np.diff(np.concatenate(([0], kept.view(np.int8), [0]))))
        for b, e in zip(edges[0::2], edges[1::2]):  # runs of kept records
            pieces.append(view[int(line_start[b]):int(line_start[e])])
        return np.frombuffer(b"".join(pieces) + b"".join(self.split_lines), dtype=np.uint8)

    def merge(self, lik: np.ndarray) -> np.ndarray:
        """Per-row class likelihoods of the scored pass (n_kept + n_split, K) -> (N, W) matrix in
        input record order, zero padded (merge_and_assign_pls, variant_filtering_utils.py:346-408,
        and the fill loop of filter_variants_pipeline.py:170-172)."""
        kept = self.kept
        n_kept = int(kept.sum())
        if lik.shape[0] != n_kept + len(self.split_lines):
            raise ValueError("scored pass returned an unexpected number of rows")
        width = max([lik.shape[1]] + [g.n_alleles * (g.n_alleles + 1) // 2 for g in self.groups if len(g.rows) > 1])
        out = np.zeros((kept.size, width), dtype=np.float64)
        out[kept, :lik.shape[1]] = lik[:n_kept]
        split = lik[n_kept:]
        for g in self.groups:
            s0 = split[g.rows[0]]
            if len(g.rows) == 1:
                out[g.origin, :s0.size] = s0
                continue
            if s0.size < 3:  # noqa: PLR2004
                raise IndexError("list index out of range")  # a 2-class model has no hom-alt likelihood to spread
            s1 = split[g.rows[1]]
            i1, i2 = g.orig_alleles.index(g.second_alleles[0]), g.orig_alleles.index(g.second_alleles[1])
            vals = [s0[0], s0[1], s0[2] * s1[0], 0.0, s0[2] * s1[1], s0[2] * s1[2]]
            where = [get_pl_idx(t) for t in ((0, 0), (0, i1), (i1, i1), (0, i2), (i1, i2), (i2, i2))]
            row = np.zeros(width)
            row[where] = vals
            out[g.origin] = row
        return out


# ------------------------------------------------------------------ the device form (csrc/multiallelic.cu)
MA_KEEP, MA_SUB_A, MA_SUB_R, MA_ERR_G, MA_ERR_NUM, MA_SPECIAL = 0, 1, 2, 3, 4, 5
_SPECIAL_INFO = ("x_ic", "x_il", "x_hil", "x_hin")


def rules_blob(plan: SplitPlan) -> bytes:
    """The per-tag rules of ``SplitPlan._rewrite`` / ``convert`` as the flat table ``ugvc_ma_set_rules`` takes: for every
    INFO / FORMAT tag of the header (lower-cased, first spelling wins, as in ``plan.rule``) what happens to its
    value in a split row -- kept, the pair's elements of a Number=A / Number=R list, an error for Number=G /
    Number=n, or replaced by a derived value (X_IC / X_IL / X_HIL / X_HIN when the loader keeps the column)."""
    header = plan.header

    def table(is_format: bool, tags) -> list:
        out, seen = [], set()
        for tag in tags:
            col = tag.lower()
            if col in seen:
                continue
            seen.add(col)
            action, number = MA_KEEP, 0
            if not is_format and col in _SPECIAL_INFO and col in plan.loaded:
                action = MA_SPECIAL + _SPECIAL_INFO.index(col)
            elif col in plan.loaded and col not in plan.SPECIAL:
                rule = plan.rule.get((is_format, col))
                if rule == "A":
                    action = MA_SUB_A
                elif rule == "R":
                    action = MA_SUB_R
                elif rule == "G":
                    action = MA_ERR_G
                elif rule is not None and rule != ".":
                    action, number = MA_ERR_NUM, int(rule) & 0xFFFF
            name = col.encode()
            if action != MA_KEEP and len(name) <= 32:  # noqa: PLR2004
                out.append(struct.pack("<32sBBH", name, len(name), action, number))
        return out

    info, fmt = table(False, header.info), table(True, header.formats)
    flags = (1 if "QD" in header.info else 0) | (2 if "GQ" in header.formats else 0)
    spell = []
    for k, col in enumerate(_SPECIAL_INFO):
        if col in plan.loaded:
            flags |= 1 << (4 + k)
        spell.append(plan.header_tag(col).encode()[:32])
    head = struct.pack("<IIII", 0x4D41524C, len(info), len(fmt), flags)
    head += b"".join(struct.pack("<32s", t) for t in spell) + bytes(len(t) for t in spell)
    return head + b"".join(info) + b"".join(fmt)


_MA_ERRORS = {
    1: (AssertionError, "One of the alleles should be present in the GT"),
    2: (RuntimeError, "Special treatment is required for 'G' fields, not supported by this function"),
    3: (RuntimeError, "Number of a per-allele tag is not supported"),
    4: (RuntimeError, "Can't deal with spanning deletion allele without the spandel"),
    5: (ValueError, "Input contains non ACGTacgt characters"),
    6: (IndexError, "list index out of range"),
    7: (TypeError, "'NoneType' object is not subscriptable"),
    8: (ValueError, "invalid literal for int() with base 10"),
    9: (RuntimeError, "a record beyond the limits of the device split (more than 32 alleles, or a malformed line)"),
    10: (IndexError, "list index out of range"),
}


class DeviceSplitPlan:
    """``SplitPlan`` on the device: same constructor, ``build`` and ``merge``; owns a ``ugvc_ma`` handle."""

    def __init__(self, header, loaded_columns: dict, ref_seq: str, device: int = 0):
        from variantcalling_b200 import lib

        self._lib = lib.load_library()
        self._UgvcError = lib.UgvcError
        self._UgvcDataError = lib.UgvcDataError
        self.host = SplitPlan(header, loaded_columns, "")  # the rule tables only (its build / merge are not used)
        self.set_reference(ref_seq)
        h = C.c_void_p()
        rc = self._lib.ugvc_ma_create(device, C.byref(h))
        if rc != 0:
            raise lib.UgvcError(rc, "ugvc_ma_create failed (no CUDA device?)")
        self.h = h
        blob = rules_blob(self.host)
        self._check(self._lib.ugvc_ma_set_rules(self.h, blob, len(blob)))
        self.kept: np.ndarray | None = None
        self.origins = np.zeros(0, dtype=np.int32)   # record of every group, in processing order
        self.n_rows = np.zeros(0, dtype=np.uint8)
        self.group_alleles = np.zeros(0, dtype=np.uint8)
        self.stats = np.zeros(8, dtype=np.int64)

    def set_reference(self, ref_seq):
        """The next contig's sequence: str, bytes or a uint8 array (the handle and its device buffers are reused from
        contig to contig)."""
        if isinstance(ref_seq, np.ndarray):
            self.ref = np.ascontiguousarray(ref_seq, dtype=np.uint8)
        else:
            self.ref = np.frombuffer(ref_seq.encode() if isinstance(ref_seq, str) else ref_seq, dtype=np.uint8)

    def close(self):
        if getattr(self, "h", None):
            self._lib.ugvc_ma_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001, S110
            pass

    def launch_count(self) -> int:
        return int(self._lib.ugvc_ma_launch_count(self.h))

    @property
    def n_scored_records(self) -> int:
        """Lines of the text the last ``build`` returned (untouched records + split rows)."""
        return int(self.stats[2] + self.stats[3])

    def _check(self, rc: int):
        if rc != 0:
            raise self._UgvcError(rc, self._lib.ugvc_ma_last_error(self.h).decode())

    def build(self, text: np.ndarray, line_start: np.ndarray, recinfo: np.ndarray) -> np.ndarray:
        """-> the text of the scored pass (``SplitPlan.build``).  The reference's failures keep their types."""
        text = np.ascontiguousarray(text, dtype=np.uint8)
        line_start = np.ascontiguousarray(line_start, dtype=np.int64)
        recinfo = np.ascontiguousarray(recinfo)
        n = int(recinfo.size)
        rc = self._lib.ugvc_ma_build(self.h, text.ctypes.data, text.size, line_start.ctypes.data, recinfo.ctypes.data, n,
                                     self.ref.ctypes.data if self.ref.size else None, self.ref.size,
                                     self.stats.ctypes.data_as(C.POINTER(C.c_int64)))
        if rc not in (0, -4):
            self._check(rc)
        self._raise_reference_failure()
        n_singles, n_cluster = int(self.stats[0]), int(self.stats[1])
        n_groups = n_singles + n_cluster
        out = np.empty(int(self.stats[4] + self.stats[5]), dtype=np.uint8)
        self.origins = np.empty(n_groups, dtype=np.int32)
        self.n_rows = np.empty(n_groups, dtype=np.uint8)
        self.group_alleles = np.empty(n_groups, dtype=np.uint8)
        self._check(self._lib.ugvc_ma_fetch(self.h, out.ctypes.data, out.size, self.origins.ctypes.data, self.n_rows.ctypes.data,
                                            self.group_alleles.ctypes.data, n_groups))
        kept = np.ones(n, dtype=bool)
        kept[self.origins] = False
        self.kept = kept
        return out

    @staticmethod
    def _raise(code: int):
        exc, msg = _MA_ERRORS.get(code, (RuntimeError, f"device split failed with code {code}"))
        raise exc(msg)

    def _raise_reference_failure(self, merge_failed: bool = False):
        """Raise what the reference raises on the contig of the last build (self.stats) or merge, in the order in which it
        meets its failures (training_prep.py:255-287, then merge_and_assign_pls); nothing when there is none."""
        n_singles, n_cluster = int(self.stats[0]), int(self.stats[1])
        err_group, err_code = -1, 0
        g, c = C.c_int64(-1), C.c_int32(0)
        if not merge_failed and self._lib.ugvc_ma_data_error(self.h, C.byref(g), C.byref(c)) == 0:
            err_group, err_code = g.value, c.value
        if n_singles == 0:
            raise ValueError("No objects to concatenate")  # pd.concat([]) in training_prep.py:261
        if 0 <= err_group < n_singles:
            self._raise(err_code)
        if n_cluster == 0:
            raise KeyError("spanning_deletion")  # variant_filtering_utils.py:339 on a frame without the column
        if err_group >= 0:
            self._raise(err_code)
        if merge_failed:
            raise IndexError("list index out of range")  # a 2-class model has no hom-alt likelihood to spread

    def filter_bgzf(self, ctx, index_ctx, bgzf, skip_head: int, take_bytes: int, threshold: float, flags: int,
                    max_records: int, **kw) -> dict | None:
        """One whole contig through the device file path with this plan's handle and reference
        (``lib.Context.filter_bgzf_split``; ``kw`` as there).  The reference's failures keep their types, as in
        ``build`` / ``merge``; the result also holds "split_stats" (``ugvc_ma_build``'s counts)."""
        try:
            res = ctx.filter_bgzf_split(bgzf, skip_head, take_bytes, threshold, flags, max_records, index_ctx=index_ctx,
                                        ma=self.h, ref=self.ref, split_stats=self.stats, **kw)
        except self._UgvcDataError:
            if self.stats[7] == 0:  # a data error of K1, not of the split
                raise
            self._raise_reference_failure(merge_failed=self.stats[7] == 2)  # noqa: PLR2004
            raise
        if res is not None:
            res["split_stats"] = self.stats.copy()
        return res

    def merge(self, lik: np.ndarray) -> np.ndarray:
        """``SplitPlan.merge``: (n_kept + n_split, K) likelihoods -> (N, W) in input record order."""
        lik = np.ascontiguousarray(lik, dtype=np.float64)
        n_rows, k = lik.shape
        if n_rows != int(self.stats[2] + self.stats[3]):
            raise ValueError("scored pass returned an unexpected number of rows")
        width = max(k, int(self.stats[6]))
        out = np.empty((int(self.kept.size), width), dtype=np.float64)
        rc = self._lib.ugvc_ma_merge(self.h, lik.ctypes.data, n_rows, k, out.ctypes.data, width)
        if rc == -4:  # noqa: PLR2004  (UGVC_E_DATA)
            self._raise_reference_failure(merge_failed=True)
        self._check(rc)
        return out


def make_split_plan(header, loaded_columns: dict, ref_seq: str, device: int = 0, reuse=None):
    """The tool's split plan: the device form (``reuse``: the plan of the previous contig, whose handle and buffers
    carry over), or the Python model of it with UGVC_MA_HOST=1 (A/B, like UGVC_K1_LEGACY)."""
    if os.environ.get("UGVC_MA_HOST", "0") not in ("", "0"):
        return SplitPlan(header, loaded_columns, ref_seq if isinstance(ref_seq, str) else bytes(ref_seq).decode())
    if isinstance(reuse, DeviceSplitPlan) and reuse.h:
        reuse.set_reference(ref_seq)
        return reuse
    return DeviceSplitPlan(header, loaded_columns, ref_seq, device)


def score_math(lik: np.ndarray, threshold: float):
    """phreds / quals / gq / low_score from the likelihood matrix (filter_variants_pipeline.py:174-180,192)."""
    phreds = -10 * np.log10(lik + 1e-10)
    quals = np.clip(30 + phreds[:, 0] - np.min(phreds[:, 1:], axis=1), 0, None)
    return phreds, quals, (quals <= threshold).astype(np.uint8)
