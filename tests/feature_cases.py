"""Edge records for the feature path: VCF text -> K1 slot words -> K2 policies -> the feature matrix K3 scores.

Each case is a clean record of one flavour with a few fields rewritten, the reducer or policy of the plan it aims at
(``target``: tag and ``RED_*`` / policy name, checked against the compiled slot table), and what the reference
transformer gives for it: the values of the named features, or ``RAISES`` when the reference refuses the record.
``slow`` marks a record the K1 tile kernel hands to the generic parser (strings longer than its 31-byte key limit,
region values).  ``tests/test_feature_cases_cpu.py`` pins every expectation on the reference side and
``tests/test_gpu_feature_edges.py`` runs the corpus through both K1 tiers and both K3 paths.

Flavours: ``ss`` (single sample, customs incl. ``long_hmer``, ``region_annotations`` and categoricals), ``ss1`` (the
same records under a header that declares the motifs and X_CSS scalar, AF ``Number=.``), ``dv`` (deep_variant), ``dvx``
(deep_variant_extended) and ``cnv``."""
from __future__ import annotations

from dataclasses import dataclass, replace

import numpy as np
import pandas as pd

from oracle import ref_pipeline as R
from oracle.vcf_reader import OracleVariantFile
from variantcalling_b200 import transformers as T
from variantcalling_b200.tprep_constants import VcfType

RAISES = "raises"
SS_CUSTOMS = ["LCR", "MAP_UNIQUE", "LONG_HMER", "UG_HCR", "EXOME", "REGION_ANNOTATIONS"]
LCR24 = "lcr_category_of_24_bytes"   # a known category at the 24-byte PlanString limit
CSS24 = "css_category_of_24_bytes"
REGIONS = ("Telomere_Centromere", "Clusters", "Coverage-Mappability")
DVX_TAGS = ["MQ0_REF", "MQ0_ALT", "LS_REF", "LS_ALT", "RS_REF", "RS_ALT", "MEAN_NM_REF", "MEDIAN_NM_REF", "MEAN_NM_ALT",
            "MEDIAN_NM_ALT", "MEAN_MIS_REF", "MEDIAN_MIS_REF", "MEAN_MIS_ALT", "MEDIAN_MIS_ALT"]
MOTIF = {"A": 1, "T": 2, "G": 3, "C": 4, "N": 5}
# htslib stores VCF Integer values as int32 and rejects a literal outside it; the oracle reader (Python int) keeps it
INT32 = "Integer literal outside int32"
# "KEY=" reaches the reference as None (imputed) for a Number=1 value and as () for a vector; the device reads an empty
# numeric value as a bad literal and an empty string as a string without a base
EMPTY = "empty numeric value"
EMPTY_STR = "empty string value"


@dataclass(frozen=True)
class Case:
    name: str
    flavour: str
    edits: tuple                 # ("info", KEY, value | None | FLAG), ("fmt", KEY, value | None), ("col", i, text), ("fmt_keep", n)
    target: tuple                # (tag or None, reducer / policy name)
    want: object                 # {feature name: value} or RAISES
    slow: bool = False
    device: object = None        # where the device differs on purpose: its result (RAISES or {feature: value}) ...
    deviation: str = ""          # ... and why

    @property
    def on_device(self):
        return self.want if self.device is None else self.device


FLAG = object()


def apply(line: str, edits) -> str:
    c = line.split("\t")
    for op in edits:
        if op[0] == "col":
            c[op[1]] = op[2]
        elif op[0] == "info":
            _, key, val = op
            kv = [] if c[7] == "." else c[7].split(";")
            at = next((i for i, x in enumerate(kv) if x.split("=", 1)[0] == key), len(kv))   # keep the key's place
            kv = [x for x in kv if x.split("=", 1)[0] != key]
            if val is FLAG:
                kv.insert(at, key)
            elif val is not None:
                kv.insert(at, f"{key}={val}")
            c[7] = ";".join(kv) if kv else "."
        elif op[0] == "fmt":
            _, key, val = op
            keys, vals = c[8].split(":"), c[9].split(":")
            if key in keys:
                i = keys.index(key)
                if val is None:
                    del keys[i], vals[i]
                else:
                    vals[i] = val
            elif val is not None:
                keys.append(key)
                vals.append(val)
            c[8], c[9] = ":".join(keys), ":".join(vals)
        elif op[0] == "fmt_keep":
            c[9] = ":".join(c[9].split(":")[: op[1]])
        else:
            raise ValueError(op)
    return "\t".join(c)


# ------------------------------------------------------------------------------------------------ flavours
def _ss_lines(n, seed):
    from tests import util

    ds = util.make_dataset(n_records=n, n_custom=5, seed=seed)
    header = [h for h in ds["header"] if not h.startswith("#CHROM")]
    header.append('##INFO=<ID=REGION_ANNOTATIONS,Number=.,Type=String,Description="region names">')
    header.append(ds["header"][-1])
    lines = list(ds["lines"])
    # categories the edge cases name: a 24-byte one for a custom categorical and for X_CSS
    for i in range(3, len(lines), 97):
        lines[i] = apply(lines[i], [("info", "LCR", LCR24), ("info", "X_CSS", CSS24)])
    return header, lines, ds["labels"]


def _rename_header(header, repl):
    out = []
    for h in header:
        for tag, new in repl.items():
            if h.startswith(f"##INFO=<ID={tag},"):
                h = new
        out.append(h)
    return out


def _dvx(n, seed):
    from tests import dv_data

    ds = dv_data.generate(n, seed=seed)
    rng = np.random.default_rng(seed)
    header = ds["header"][:-1]
    for t in DVX_TAGS:
        typ = "Float" if t.startswith(("MEAN", "MEDIAN")) else "Integer"
        header.append(f'##INFO=<ID={t},Number=1,Type={typ},Description="{t}">')
    header.append(ds["header"][-1])
    lines = []
    for ln in ds["lines"]:
        c = ln.split("\t")
        add = []
        for t in DVX_TAGS:
            if rng.random() < 0.85:
                add.append(f"{t}={rng.uniform(0, 9):.3f}" if t.startswith(("MEAN", "MEDIAN")) else f"{t}={int(rng.integers(0, 40))}")
        c[7] = ";".join([c[7], *add]) if add else c[7]
        lines.append("\t".join(c))
    return header, lines, ds["labels"], ds["customs"]


def flavour(name: str, n: int = 400, seed: int = 41) -> dict:
    """-> dict(header=[lines], lines=[clean records], labels, customs, vtype)."""
    if name in ("ss", "ss1"):
        header, lines, labels = _ss_lines(n, seed)
        if name == "ss1":
            header = _rename_header(header, {
                "X_LM": '##INFO=<ID=X_LM,Number=1,Type=String,Description="left motif">',
                "X_RM": '##INFO=<ID=X_RM,Number=1,Type=String,Description="right motif">',
                "X_CSS": '##INFO=<ID=X_CSS,Number=.,Type=String,Description="cycle skip">',
                "AF": '##INFO=<ID=AF,Number=.,Type=Float,Description="allele frequency">'})
        return dict(header=header, lines=lines, labels=labels, customs=list(SS_CUSTOMS), vtype=VcfType.SINGLE_SAMPLE)
    if name == "dv":
        from tests import dv_data

        ds = dv_data.generate(n, seed=seed)
        return dict(header=ds["header"], lines=ds["lines"], labels=ds["labels"], customs=ds["customs"], vtype=VcfType.DEEP_VARIANT)
    if name == "dvx":
        header, lines, labels, customs = _dvx(n, seed)
        return dict(header=header, lines=lines, labels=labels, customs=customs + DVX_TAGS,
                    annots=[c.lower() for c in customs], vtype=VcfType.DEEP_VARIANT_WITH_SOFTCLIP_COUNTS)
    if name == "cnv":
        from tests.test_gpu_cnv import CUSTOM, make_cnv_vcf

        header, lines = make_cnv_vcf(n, seed)
        x = reference_matrix(dict(header=header, customs=CUSTOM), lines, transformer=None, vtype=VcfType.CNV)[1]
        labels = (x[:, 1] + x[:, 16] > 5).astype(int)
        return dict(header=header, lines=lines, labels=labels, customs=list(CUSTOM), vtype=VcfType.CNV)
    raise ValueError(name)


def transformer_annots(fl: dict) -> list:
    if fl["vtype"] == VcfType.CNV:
        return ["region_annotations"]
    return fl.get("annots") or [c.lower() for c in fl["customs"]]


def reference_matrix(fl: dict, lines, transformer=None, vtype=None, n_features=None):
    """The reference's feature matrix of ``lines``: the oracle reader's frame through the transformer (fitted here when
    ``transformer`` is None), fp64 -> fp32.  Raises where the reference raises: in the reader, the transformer, the
    null check of ``_validate_data``, or the input check on a value that is infinite in float32.
    -> (transformer, fp64 matrix, fp32 matrix)."""
    text = ("\n".join(fl["header"]) + "\n" + "\n".join(lines) + "\n").encode()
    df = R.harness_float_columns(R.get_vcf_df(OracleVariantFile(text), None, fl["customs"]))
    with pd.option_context("future.infer_string", False):
        if transformer is None:
            transformer = T.get_transformer(vtype or fl["vtype"], transformer_annots(fl) if vtype is None else ["region_annotations"])
            x = transformer.fit_transform(df)
        else:
            x = transformer.transform(df)
            n_features = sum(s.stop - s.start for s in transformer.output_indices_.values())
    R.validate_data(x)
    x = x.to_numpy(dtype=np.float64)
    if n_features is not None and x.shape[1] != n_features:   # the model's own check, e.g. PL wider than fitted
        raise ValueError(f"X has {x.shape[1]} features, but the model is expecting {n_features} features as input")
    with np.errstate(over="ignore"):
        x32 = x.astype(np.float32)
    if not np.isfinite(x32).all():
        raise ValueError("Input X contains infinity or a value too large for dtype('float32').")
    return transformer, x, x32


def base_record(fl: dict) -> str:
    """The clean record every case of the flavour edits: a biallelic SNP with every key the edits name."""
    for ln in fl["lines"]:
        c = ln.split("\t")
        if fl["vtype"] == VcfType.CNV:
            return ln
        if len(c[3]) == 1 and len(c[4]) == 1 and c[5] != "." and "X_IC=" in c[7]:
            return ln
    raise AssertionError("no base record")


# ------------------------------------------------------------------------------------------------ motifs
def motif_value(s: str, left: bool) -> int:
    items = reversed(s) if left else s
    acc = 0
    for ch in items:
        acc = acc * 10 + MOTIF.get(ch, 0)
    return acc


def near_f32_midpoint(n: int = 17, ulps: int = 4):
    """A motif of ``n`` bases whose exact integer value lies within ``ulps`` fp64 ulps of a float32 rounding midpoint, so
    that an accumulation that rounds a running value to fp32, or rounds differently in fp64, lands on the other side.
    Depth-first over the digits, most significant first, keeping the prefixes whose reachable values still come that
    close to a midpoint.  -> (motif read left to right, exact value)."""
    code = {1: "A", 2: "T", 3: "G", 4: "C", 5: "N"}

    def near(lo, hi):
        k = lo.bit_length() - 1
        if k != hi.bit_length() - 1:
            return True
        s, u = 1 << (k - 23), 1 << max(0, k - 52)
        a, b = lo - ulps * u, hi + ulps * u
        j = -((s - 2 * a) // (2 * s))       # the first midpoint (j + 1/2) s at or above a
        return (2 * j + 1) * s <= 2 * b

    stack = [(0, n)]
    while stack:
        p, r = stack.pop()
        if r == 0:
            return "".join(code[int(d)] for d in str(p)), p
        for d in range(1, 6):
            q = p * 10 + d
            if near(q * 10 ** (r - 1) + int("1" * (r - 1) or 0), q * 10 ** (r - 1) + int("5" * (r - 1) or 0)):
                stack.append((q, r - 1))
    raise AssertionError("no motif")


MID_MOTIF, MID_VALUE = near_f32_midpoint()


def f32(v) -> float:
    return float(np.float32(v))


# ------------------------------------------------------------------------------------------------ the corpus
def _ss_cases():
    out = []

    def add(name, edits, target, want, slow=False, fl="ss"):
        out.append(Case(name, fl, tuple(edits), target, want, slow))

    # ---- RED_NUM: integers (DP is INFO and FORMAT Integer Number=1, imputed with 0; GQ FORMAT only)
    for s, v in (("2147483647", 2147483647), ("-2147483647", -2147483647), ("0", 0), ("-0", 0), ("+5", 5), ("007", 7)):
        add(f"int_gq_{s}", [("fmt", "GQ", s)], ("GQ", "RED_NUM"), {"gq": f32(v)})
    for s in ("2147483648", "-2147483649", "99999999999"):
        out.append(Case(f"int_gq_beyond_int32_{s}", "ss", (("fmt", "GQ", s),), ("GQ", "RED_NUM"), {"gq": f32(int(s))},
                        device=RAISES, deviation=INT32))
    for s in ("1e", "1.5", "5x", "0x10"):
        add(f"int_gq_bad_{s}", [("fmt", "GQ", s)], ("GQ", "RED_NUM"), RAISES)
    add("int_gq_dot", [("fmt", "GQ", ".")], ("GQ", "RED_NUM"), {"gq": 0.0})
    add("int_gq_absent", [("fmt", "GQ", None)], ("GQ", "POL_VALUE absent"), {"gq": 0.0})
    add("fmt_dp_overrides_info", [("info", "DP", "5"), ("fmt", "DP", "7")], ("DP", "RED_NUM"), {"dp": 7.0})
    add("fmt_dp_dot_overrides_info", [("info", "DP", "5"), ("fmt", "DP", ".")], ("DP", "RED_NUM"), {"dp": 0.0})
    add("info_dp_only", [("info", "DP", "5"), ("fmt", "DP", None)], ("DP", "RED_NUM"), {"dp": 5.0})
    add("trailing_fmt_dropped", [("fmt_keep", 2)], ("PL", "POL_VALUE missing"),
        {"gq": 0.0, "pl_0": 1000.0, "pl_1": 1000.0, "pl_2": 1000.0})
    # ---- RED_NUM: floats (SOR imputed, MQ imputed, QD imputed, AF first element of Number=A)
    for s in ("1e", "nan5", "1.5.2", "--1"):
        add(f"float_bad_{s}", [("info", "SOR", s)], ("SOR", "RED_NUM"), RAISES)
    for s, v in (("-0", -0.0), ("+2.5", 2.5), ("000123.4500", 123.45), ("3.4028234e38", 3.4028234e38),
                 ("1e-46", 0.0), ("16777217", 16777217.0)):
        add(f"float_sor_{s}", [("info", "SOR", s)], ("SOR", "RED_NUM"), {"sor": f32(v)})
    add("float_sor_dot", [("info", "SOR", ".")], ("SOR", "RED_NUM"), {"sor": 0.0})
    out.append(Case("float_sor_empty", "ss", (("info", "SOR", ""),), ("SOR", "RED_NUM"), {"sor": 0.0}, device=RAISES,
                    deviation=EMPTY))
    for s in ("3.5e38", "1e39", "-1e39", "inf", "-inf", "Infinity"):
        add(f"float_sor_overflow_{s}", [("info", "SOR", s)], ("SOR", "RED_NUM"), RAISES)
    add("float_sor_nan", [("info", "SOR", "nan")], ("SOR", "RED_NUM"), {"sor": 0.0})    # NaN is imputed
    add("af_dot_element", [("info", "AF", ".")], ("AF", "POL_ERROR missing"), RAISES)
    add("af_two_elements", [("info", "AF", "0.25,0.5")], ("AF", "RED_NUM"), {"af": 0.25})
    add("af_absent", [("info", "AF", None)], ("AF", "POL_VALUE absent"), {"af": 0.0})
    # ---- vectors against the fitted width (PL: width 3, 1000 for a short vector or a '.' element)
    add("pl_width", [("fmt", "PL", "0,10,20")], ("PL", "RED_NUM"), {"pl_0": 0.0, "pl_1": 10.0, "pl_2": 20.0})
    add("pl_short", [("fmt", "PL", "0,10")], ("PL", "RED_NUM"), {"pl_0": 0.0, "pl_1": 10.0, "pl_2": 1000.0})
    add("pl_dot_elements", [("fmt", "PL", "0,.,20")], ("PL", "RED_NUM"), {"pl_0": 0.0, "pl_1": 1000.0, "pl_2": 20.0})
    add("pl_width_plus_one", [("fmt", "PL", "0,10,20,30")], ("PL", "RED_LEN"), RAISES)
    add("pl_absent", [("fmt", "PL", None)], ("PL", "RED_NUM"), {"pl_0": 1000.0, "pl_1": 1000.0, "pl_2": 1000.0})
    add("ad_one_element", [("fmt", "AD", "4")], ("AD", "RED_NUM"), RAISES)                  # ragged doublet
    add("ad_three_elements", [("fmt", "AD", "4,5,6")], ("AD", "RED_NUM"), {"ad_0": 4.0, "ad_1": 5.0})
    add("mq0c_dot_element", [("info", "MQ0C", "3,.")], ("MQ0C", "RED_NUM"), RAISES)
    # ---- RED_GT_HOM
    for s, v in (("1/1", 1.0), ("1|1", 1.0), ("1/1/1", 0.0), ("1/", 0.0), ("11", 0.0), ("0/1", 0.0), ("./.", 0.0),
                 ("1/2", 0.0), ("2/2", 0.0), ("1", 0.0), ("1/10", 0.0), (".", 0.0)):
        add(f"gt_{s}", [("fmt", "GT", s)], ("GT", "RED_GT_HOM"), {"gt": v})
    # ---- RED_BASE (X_HIN: first element of a Number=A string)
    for s, v in (("A", 1.0), ("T", 2.0), ("G", 3.0), ("C", 4.0), ("N", 0.0), ("a", 0.0), ("AC", 0.0), (".", 0.0),
                 ("G,A", 3.0), ("GA,A", 0.0)):
        add(f"base_x_hin_{s or 'empty'}", [("info", "X_HIN", s)], ("X_HIN", "RED_BASE"), {"x_hin": v})
    out.append(Case("base_x_hin_empty", "ss", (("info", "X_HIN", ""),), ("X_HIN", "RED_BASE"), RAISES, device={"x_hin": 0.0},
                    deviation=EMPTY_STR))                                                # () has no first element
    add("base_x_hin_32_bytes", [("info", "X_HIN", "A" * 32)], ("X_HIN", "RED_BASE"), {"x_hin": 0.0})   # a long key: 0
    # ---- RED_INSDEL (X_IC)
    for s, v in (("ins", -1.0), ("del", 1.0), ("NA", 0.0), ("ins,del", -1.0)):
        add(f"insdel_{s}", [("info", "X_IC", s)], ("X_IC", "RED_INSDEL"), {"x_ic": v})
    for s in ("in", "insx", "de", "dell", "N", "NAA", "INS", "Del", "na", ".", ""):
        add(f"insdel_bad_{s or 'empty'}", [("info", "X_IC", s)], ("X_IC", "RED_INSDEL"), RAISES)
    # ---- RED_MOTIF_L / R on a Number=A tuple: only one-character elements count
    for s, lv in (("A", 1), ("C,G", 34), ("CG,A", 10), ("N,a", 5), ("", 0), (".", 0)):
        rv = motif_value([x if len(x) == 1 else "" for x in s.split(",")] if s else [], False)
        add(f"motif_tuple_{s or 'empty'}", [("info", "X_LM", s), ("info", "X_RM", s)], ("X_LM", "RED_MOTIF_L"),
            {"x_lm": f32(lv), "x_rm": f32(rv)})
    # ---- dictionaries: X_CSS (Number=A, OrdinalEncoder), LCR (custom categorical, FALSE when absent)
    add("css_known", [("info", "X_CSS", "cycle-skip")], ("X_CSS", "RED_DICT"), {"x_css": ("cat", "cycle-skip")})
    add("css_24_bytes", [("info", "X_CSS", CSS24)], ("X_CSS", "RED_DICT"), {"x_css": ("cat", CSS24)})
    add("css_unknown", [("info", "X_CSS", "skip")], ("X_CSS", "RED_DICT"), RAISES)
    add("css_24_bytes_plus_one", [("info", "X_CSS", CSS24 + "x")], ("X_CSS", "RED_DICT"), RAISES)
    add("css_32_bytes", [("info", "X_CSS", "c" * 32)], ("X_CSS", "RED_DICT"), RAISES, slow=True)
    add("css_dot", [("info", "X_CSS", ".")], ("X_CSS", "RED_DICT"), RAISES)
    add("lcr_known", [("info", "LCR", "TRUE")], ("LCR", "RED_DICT"), {"lcr": ("cat", "TRUE")})
    add("lcr_24_bytes", [("info", "LCR", LCR24)], ("LCR", "RED_DICT"), {"lcr": ("cat", LCR24)})
    add("lcr_absent", [("info", "LCR", None)], ("LCR", "POL_VALUE absent"), {"lcr": ("cat", "FALSE")})
    add("lcr_prefix", [("info", "LCR", LCR24[:23])], ("LCR", "RED_DICT"), RAISES)
    add("lcr_unknown", [("info", "LCR", "MAYBE")], ("LCR", "RED_DICT"), RAISES)
    add("lcr_31_bytes", [("info", "LCR", "L" * 31)], ("LCR", "RED_DICT"), RAISES)
    add("lcr_32_bytes", [("info", "LCR", "L" * 32)], ("LCR", "RED_DICT"), RAISES, slow=True)
    add("lcr_dot", [("info", "LCR", ".")], ("LCR", "RED_DICT"), RAISES)
    # ---- RED_STRNUM (long_hmer: None -> "0", then pd.to_numeric)
    for s, v in (("7", 7), ("+5", 5), ("-0.0", -0.0), ("007", 7), ("5.", 5), (".5", 0.5),
                 ("12345678901234567890", 12345678901234567890), (" 5", 5), ("5 ", 5), ("  -2.5 ", -2.5), ("1e3", 1000.0)):
        add(f"strnum_{s!r}", [("info", "LONG_HMER", s)], ("LONG_HMER", "RED_STRNUM"), {"long_hmer": f32(v)}, slow=" " in s)
    add("strnum_absent", [("info", "LONG_HMER", None)], ("LONG_HMER", "POL_VALUE absent"), {"long_hmer": 0.0})
    out.append(Case("strnum_empty", "ss", (("info", "LONG_HMER", ""),), ("LONG_HMER", "POL_VALUE absent"), {"long_hmer": 0.0},
                    device=RAISES, deviation=EMPTY))
    for s in (".", "1_000", "0x10", "nan", "NaN", "inf", "-inf", "1e400", "1e", "5,6", " ", "1 2"):
        add(f"strnum_bad_{s!r}", [("info", "LONG_HMER", s)], ("LONG_HMER", "RED_STRNUM"), RAISES)
    # ---- RED_REGION (Number=. tuple of names; absent -> 0)
    names = sorted(REGIONS)
    enc = T._get_region_encoding()  # noqa: SLF001
    for mask in range(1, 8):
        sub = [nm for i, nm in enumerate(names) if mask >> i & 1]
        val = ",".join(reversed(sub))
        add(f"region_{mask}", [("info", "REGION_ANNOTATIONS", val)], ("REGION_ANNOTATIONS", "RED_REGION"),
            {"region_annotations": float(enc[tuple(sub)])}, slow=True)
    add("region_absent", [("info", "REGION_ANNOTATIONS", None)], ("REGION_ANNOTATIONS", "POL_VALUE absent"),
        {"region_annotations": 0.0})
    add("region_repeated", [("info", "REGION_ANNOTATIONS", "Clusters,Clusters")], ("REGION_ANNOTATIONS", "RED_REGION"),
        RAISES, slow=True)
    add("region_unknown", [("info", "REGION_ANNOTATIONS", "Exome")], ("REGION_ANNOTATIONS", "RED_REGION"), RAISES, slow=True)
    add("region_dot", [("info", "REGION_ANNOTATIONS", ".")], ("REGION_ANNOTATIONS", "RED_REGION"), RAISES, slow=True)
    # ---- fixed columns
    add("qual_dot", [("col", 5, ".")], (None, "RED_FIX_QUAL"), RAISES)
    add("qual_overflow", [("col", 5, "3.5e38")], (None, "RED_FIX_QUAL"), RAISES)
    add("qual_max_float32", [("col", 5, "3.4028234e38")], (None, "RED_FIX_QUAL"), {"qual": f32(3.4028234e38)})
    add("alt_dot", [("col", 4, ".")], (None, "RED_FIX_ALLELE1"), RAISES)
    add("alt_multi", [("col", 4, "C,T"), ("fmt", "AD", "1,2,3"), ("fmt", "PL", "0,1,2")], (None, "RED_FIX_ALLELE1"),
        {"alleles_1": 4.0, "indel": 0.0, "ad_1": 2.0})
    add("ref_alt_unequal", [("col", 3, "A"), ("col", 4, "AT")], (None, "RED_FIX_INDEL"),
        {"indel": 1.0, "alleles_0": 1.0, "alleles_1": 0.0})
    add("ref_alt_multi_unequal", [("col", 3, "A"), ("col", 4, "G,AT"), ("fmt", "AD", "1,2,3"), ("fmt", "PL", "0,1,2")],
        (None, "RED_FIX_INDEL"), {"indel": 1.0, "alleles_1": 3.0})
    add("ref_lower_case", [("col", 3, "a"), ("col", 4, "c")], (None, "RED_FIX_ALLELE0"), {"alleles_0": 0.0, "alleles_1": 0.0})

    # ---- ss1: scalar motifs (string characters), X_CSS Number=., AF Number=.
    def motif(name, s):
        target = ("X_RM", "RED_MOTIF_R") if "right" in name else ("X_LM", "RED_MOTIF_L")
        add(f"motif_{name}", [("info", "X_LM", s), ("info", "X_RM", s)], target,
            {"x_lm": f32(motif_value(s, True)), "x_rm": f32(motif_value(s, False))}, slow=len(s) > 31, fl="ss1")

    out.append(Case("motif_empty", "ss1", (("info", "X_LM", ""), ("info", "X_RM", "")), ("X_LM", "RED_MOTIF_L"), RAISES,
                    device={"x_lm": 0.0, "x_rm": 0.0}, deviation=EMPTY_STR))            # list(None)
    for s in ("ACGTN", "acgtn", "A", ".", "AXC", "NNNNN", "A,C"):
        motif(repr(s), s)
    rng = np.random.default_rng(7)
    for n in (5, 16, 17, 31, 32, 39, 40):
        s = "".join("ACGT"[int(d)] for d in rng.integers(0, 4, size=n))
        if n < 39:
            motif(f"len{n}", s)
        else:   # > 3.4e38 in float32: the input check refuses the record
            add(f"motif_len{n}", [("info", "X_LM", s), ("info", "X_RM", s)], ("X_LM", "RED_MOTIF_L"), RAISES, slow=True,
                fl="ss1")
    motif("len16_ccccc", "C" * 16)
    motif("len17_ccccc", "C" * 17)
    motif("near_f32_midpoint_right", MID_MOTIF)
    motif("near_f32_midpoint_left", MID_MOTIF[::-1])
    add("css_scalar_known", [("info", "X_CSS", "cycle-skip")], ("X_CSS", "RED_DICT"), {"x_css": ("cat", "cycle-skip")}, fl="ss1")
    add("css_scalar_tuple", [("info", "X_CSS", "cycle-skip,weird")], ("X_CSS", "RED_DICT"), {"x_css": ("cat", "cycle-skip")}, fl="ss1")
    add("af_dot_number_dot", [("info", "AF", ".")], ("AF", "POL_ERROR missing"), RAISES, fl="ss1")
    add("af_number_dot", [("info", "AF", "0.125,7")], ("AF", "RED_NUM"), {"af": 0.125}, fl="ss1")
    return out


def _dv_cases():
    out = []
    out += [Case("dv_vaf_dot", "dv", (("fmt", "VAF", "."),), ("VAF", "POL_ERROR missing"), RAISES),
            Case("dv_vaf_two", "dv", (("fmt", "VAF", "0.25,0.5"),), ("VAF", "RED_NUM"), {"vaf": 0.25})]
    for fl in ("dv", "dvx"):
        out += [Case(f"{fl}_gt_hom", fl, (("fmt", "GT", "1|1"),), ("GT", "RED_GT_HOM"), {"gt": 1.0}),
                Case(f"{fl}_gq_dot", fl, (("fmt", "GQ", "."),), ("GQ", "RED_NUM"), {"gq": 0.0}),
                Case(f"{fl}_pl_short", fl, (("fmt", "PL", "5"),), ("PL", "RED_NUM"), {"pl_0": 5.0, "pl_1": 1000.0, "pl_2": 1000.0}),
                Case(f"{fl}_long_hmer_space", fl, (("info", "LONG_HMER", " 9"),), ("LONG_HMER", "RED_STRNUM"), {"long_hmer": 9.0},
                     slow=True)]
    if True:
        fl = "dvx"
        out += [Case("dvx_mq0_ref_absent", fl, (("info", "MQ0_REF", None),), ("MQ0_REF", "POL_VALUE absent"), {"mq0_ref": 0.0}),
                Case("dvx_mq0_ref_dot", fl, (("info", "MQ0_REF", "."),), ("MQ0_REF", "RED_NUM"), {"mq0_ref": 0.0}),
                Case("dvx_mq0_ref_max", fl, (("info", "MQ0_REF", "2147483647"),), ("MQ0_REF", "RED_NUM"), {"mq0_ref": f32(2**31 - 1)}),
                Case("dvx_mq0_ref_over", fl, (("info", "MQ0_REF", "2147483648"),), ("MQ0_REF", "RED_NUM"), {"mq0_ref": f32(2**31)},
                     device=RAISES, deviation=INT32),
                Case("dvx_mean_nm_alt", fl, (("info", "MEAN_NM_ALT", "1.00000006"),), ("MEAN_NM_ALT", "RED_NUM"),
                     {"mean_nm_alt": f32(1.00000006)}),
                Case("dvx_median_mis_ref_bad", fl, (("info", "MEDIAN_MIS_REF", "x"),), ("MEDIAN_MIS_REF", "RED_NUM"), RAISES)]
    return out


def _cnv_cases():
    out = []

    def add(name, edits, target, want, slow=False):
        out.append(Case(name, "cnv", tuple(edits), target, want, slow))

    add("cn_both", [("fmt", "CN", "3"), ("info", "CopyNumber", "2.5")], ("CN", "combine"), {"copynumber": 3.0})
    add("cn_info_larger", [("fmt", "CN", "1"), ("info", "CopyNumber", "2.5")], ("CN", "combine"), {"copynumber": 2.5})
    add("cn_fmt_absent", [("fmt", "CN", None), ("info", "CopyNumber", "2.5")], ("CN", "combine"), {"copynumber": 2.5})
    add("cn_fmt_dot", [("fmt", "CN", "."), ("info", "CopyNumber", "2.5")], ("CN", "combine"), {"copynumber": 2.5})
    add("cn_info_absent", [("fmt", "CN", "4"), ("info", "CopyNumber", None)], ("CopyNumber", "combine"), {"copynumber": 4.0})
    add("cn_info_dot", [("fmt", "CN", "4"), ("info", "CopyNumber", ".")], ("CopyNumber", "combine"), {"copynumber": 4.0})
    add("cn_neg", [("fmt", "CN", "-4"), ("info", "CopyNumber", "-5.5")], ("CN", "combine"), {"copynumber": -4.0})
    add("cn_both_absent", [("fmt", "CN", None), ("info", "CopyNumber", None)], ("CN", "POL_NULL"), RAISES)
    add("cn_both_dot", [("fmt", "CN", "."), ("info", "CopyNumber", ".")], ("CN", "POL_NULL"), RAISES)
    add("cn_fmt_error", [("fmt", "CN", "x"), ("info", "CopyNumber", "2.5")], ("CN", "combine"), RAISES)
    add("cn_info_error", [("fmt", "CN", "3"), ("info", "CopyNumber", "2.5.1")], ("CopyNumber", "combine"), RAISES)
    add("cn_info_overflow", [("fmt", "CN", "3"), ("info", "CopyNumber", "1e39")], ("CopyNumber", "combine"), RAISES)
    add("svtype_unknown", [("info", "SVTYPE", "INV")], ("SVTYPE", "RED_DICT"), RAISES)
    add("cnv_source_two", [("info", "CNV_SOURCE", "cn.mops,cnvpytor")], ("CNV_SOURCE", "RED_LEN"), RAISES)
    add("cnv_source_empty", [("info", "CNV_SOURCE", "")], ("CNV_SOURCE", "RED_LEN"), RAISES)
    add("region_cnv_all", [("info", "REGION_ANNOTATIONS", ",".join(REGIONS))], ("REGION_ANNOTATIONS", "RED_REGION"),
        {"region_annotations": 8.0}, slow=True)
    add("svlen_dot", [("info", "SVLEN", ".")], ("SVLEN", "POL_ERROR missing"), RAISES)
    out.append(Case("jalign_overflow", "cnv", (("info", "JALIGN_DUP_SUPPORT", "-2147483649"),), ("JALIGN_DUP_SUPPORT", "RED_NUM"),
                    {"jalign_dup_support": f32(-2147483649)}, device=RAISES, deviation=INT32))
    return out


# The tile kernel also hands over numeric literals outside its short decoder (a '+', an exponent, nan, more than eight
# characters) and records whose FORMAT keys differ from the learned order.
HANDED_OVER = {"int_gq_2147483647", "int_gq_-2147483647", "int_gq_+5", "int_gq_absent", "info_dp_only", "trailing_fmt_dropped",
               "float_sor_+2.5", "float_sor_000123.4500", "float_sor_3.4028234e38", "float_sor_1e-46", "float_sor_nan",
               "pl_absent", "strnum_'+5'", "strnum_'5.'", "strnum_'.5'", "strnum_'12345678901234567890'", "strnum_'1e3'",
               "qual_max_float32"}
CASES = [replace(c, slow=True) if c.name in HANDED_OVER else c for c in _ss_cases() + _dv_cases() + _cnv_cases()]
FLAVOURS = ("ss", "ss1", "dv", "dvx", "cnv")


def cases_of(fl: str) -> list:
    return [c for c in CASES if c.flavour == fl]


# ------------------------------------------------------------------------------------------------ plan slot table
REDUCERS = ["RED_NUM", "RED_BASE", "RED_INSDEL", "RED_DICT", "RED_MOTIF_L", "RED_MOTIF_R", "RED_STRNUM", "RED_GT_HOM",
            "RED_LEN", "RED_REGION"]
FIXED = {16: "RED_FIX_QUAL", 17: "RED_FIX_ALLELE0", 18: "RED_FIX_ALLELE1", 19: "RED_FIX_INDEL", 20: "RED_FIX_NALLELES"}
POLICIES = ["POL_VALUE", "POL_ERROR", "POL_NULL"]


def plan_tables(plan):
    """Decode the compiled plan's slot, feature and combine records (plan.h) -> dict(slots=[(tag | None, elem, RED_*)],
    features=[(slot, absent POL_*, missing POL_*)], combine_slots=[slot])."""
    import struct

    blob = plan.blob
    hdr = struct.unpack_from("<15I2H", blob, 0)
    n_tags, n_slots, n_feat, n_dicts, n_strings = hdr[2:7]
    n_checks, n_combines = hdr[15], hdr[16]

    def pad(n):
        return (n + 7) & ~7

    off = 96 + pad(40 * n_tags)
    slots = []
    for i in range(n_slots):
        tag, elem, red, _d = struct.unpack_from("<4B", blob, off + 4 * i)
        slots.append((None if tag == 0xFF else plan.tags[tag], elem, FIXED.get(red) or REDUCERS[red]))
    off += pad(4 * n_slots) + pad(4 * n_dicts) + pad(32 * n_strings)
    feats = []
    for i in range(n_feat):
        s, a, m, _av, _mv = struct.unpack_from("<HBBff", blob, off + 12 * i)
        feats.append((s, POLICIES[a], POLICIES[m]))
    off += pad(12 * n_feat) + pad(8 * n_checks)
    combines = [struct.unpack_from("<HHB3x", blob, off + 8 * i)[1] for i in range(n_combines)]
    return dict(slots=slots, features=feats, combine_slots=combines)


def reaches(plan, target) -> bool:
    """Does the plan route ``target`` = (tag | None, what) through a slot or policy of that kind?"""
    t = plan_tables(plan)
    tag, what = target
    slots_of_tag = [i for i, s in enumerate(t["slots"]) if s[0] == tag]
    if what.startswith("RED_"):
        return any(t["slots"][i][2] == what for i in slots_of_tag) or (tag is None and what in [s[2] for s in t["slots"]])
    if what == "combine":
        feat_slots = {f[0] for f in t["features"]}
        return any(i in t["combine_slots"] for i in slots_of_tag) or any(
            i in feat_slots and t["features"][[f[0] for f in t["features"]].index(i)][2] == "POL_NULL" for i in slots_of_tag)
    pol, _, which = what.partition(" ")
    idx = 1 if which == "absent" else 2
    return any(f[0] in slots_of_tag and (f[idx] == pol if which else pol in f[1:]) for f in t["features"])
