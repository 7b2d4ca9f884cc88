"""CPU: the reference side of the feature edge corpus (tests/feature_cases.py).  Every case runs through the oracle
reader and the transformer mirror, as the parity tests do, and must give the row its case states or raise; every case
must reach the reducer or policy it names in the compiled plan.  The third-party behaviour the expectations rest on
is pinned here, so a dependency change shows up as a failure of this file rather than as a silent parity drift."""
from fractions import Fraction
from functools import lru_cache

import numpy as np
import pandas as pd
import pytest

from tests import feature_cases as FC
from tests import util
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200 import transformers as T
from variantcalling_b200.vcf_header import VcfHeader


@lru_cache(maxsize=None)
def fitted(name):
    fl = FC.flavour(name)
    tr, x, _ = FC.reference_matrix(fl, fl["lines"])
    plan = MC.compile_plan(VcfHeader("\n".join(fl["header"]) + "\n"), tr, util.fit_model("lr", x, fl["labels"]), fl["customs"])
    return fl, tr, plan


def _to_numeric(s):
    return pd.to_numeric(pd.Series([s], dtype=object)).iloc[0]


@pytest.mark.parametrize("text,value", [(" 5", 5), ("5 ", 5), (" 5 ", 5), ("\t5", 5), ("+5", 5), ("007", 7), ("5.", 5.0),
                                        (".5", 0.5), ("inf", np.inf), ("-inf", -np.inf), ("Infinity", np.inf),
                                        ("1e400", np.inf), ("12345678901234567890", 12345678901234567890)])
def test_pandas_to_numeric_accepts(text, value):
    """long_hmer's convert_to_numeric (transformers.py:326-327): surrounding whitespace is ignored, inf parses."""
    assert _to_numeric(text) == value


@pytest.mark.parametrize("text", [".", "1_000", "0x10", "nan", "NaN", "-nan", "1e", "1,000", " ", "1 2"])
def test_pandas_to_numeric_refuses(text):
    with pytest.raises(ValueError, match="Unable to parse string"):
        _to_numeric(text)


def test_reader_and_imputer_facts():
    """An empty Number=1 String value reaches the transformer as None (imputed "0"), "." as the string "."."""
    from oracle.vcf_reader import typed_value

    assert typed_value("", "1", "String") is None and typed_value(".", "1", "String") == "."
    assert typed_value("", ".", "String") == () and typed_value("a,bc", "A", "String") == ("a", "bc")
    assert T.motif_encode_left(("CG", "A")) == 10 and T.motif_encode_right("ACGTN") == 14325
    assert T.region_annotation_encode(()) == 1 and T.region_annotation_encode(None) == 0


def test_the_motif_near_a_float32_midpoint():
    """The corpus motif's exact value lies within 4 fp64 ulps of a float32 rounding midpoint: an fp32 accumulation (or
    a rounding of the running value to fp32) changes its feature."""
    v = FC.MID_VALUE
    assert FC.motif_value(FC.MID_MOTIF, left=False) == v and len(FC.MID_MOTIF) >= 17
    f = np.float32(v)
    g = np.nextafter(f, np.float32(np.inf) if int(f) < v else np.float32(0))
    mid = (Fraction(int(f)) + Fraction(int(g))) / 2
    assert abs(Fraction(v) - mid) <= 4 * Fraction(int(np.spacing(float(v))))
    acc = np.float32(0)
    for ch in FC.MID_MOTIF:
        acc = np.float32(acc * np.float32(10) + np.float32(FC.MOTIF[ch]))
    assert acc != f, "the fp32 accumulation must land elsewhere for the motif to catch it"


@pytest.mark.parametrize("case", FC.CASES, ids=[c.name for c in FC.CASES])
def test_case_reaches_its_target(case):
    _, _, plan = fitted(case.flavour)
    assert FC.reaches(plan, case.target), (case.target, FC.plan_tables(plan)["slots"])


@pytest.mark.parametrize("case", FC.CASES, ids=[c.name for c in FC.CASES])
def test_reference_result(case):
    fl, tr, plan = fitted(case.flavour)
    clean = fl["lines"][:30]
    line = FC.apply(FC.base_record(fl), case.edits)
    if case.want == FC.RAISES:
        FC.reference_matrix(fl, clean, tr)  # the batch without the case is fine
        with pytest.raises((ValueError, KeyError, AssertionError, TypeError, IndexError)):
            FC.reference_matrix(fl, clean + [line], tr)
        return
    _, x64, x32 = FC.reference_matrix(fl, clean + [line], tr)
    names = plan.feature_names
    cats = {name: list(t.steps[-1][1].categories_[0]) for name, t, _ in tr.transformers_ if hasattr(t, "steps")
            and hasattr(t.steps[-1][1], "categories_")}
    for feat, want in case.want.items():
        if isinstance(want, tuple):
            want = float(cats[feat].index(want[1]))
        got = x32[-1, names.index(feat)]
        assert got.tobytes() == np.float32(want).tobytes(), (feat, got, want)


def test_compiler_refuses_a_25_byte_category_by_name():
    fl = FC.flavour("ss")
    long = FC.LCR24 + "x"
    lines = [FC.apply(ln, [("info", "LCR", long)]) if i % 50 == 7 else ln for i, ln in enumerate(fl["lines"])]
    tr, x, _ = FC.reference_matrix(fl, lines)
    with pytest.raises(MC.PlanError, match=f"category string '{long}' longer than 24 bytes"):
        MC.compile_plan(VcfHeader("\n".join(fl["header"]) + "\n"), tr, util.fit_model("lr", x, fl["labels"]), fl["customs"])


def test_compiler_refuses_a_scalar_region_tag():
    fl, tr, _ = fitted("ss")
    hdr = [h.replace("ID=REGION_ANNOTATIONS,Number=.", "ID=REGION_ANNOTATIONS,Number=1") for h in fl["header"]]
    x = np.zeros((4, len(fitted("ss")[2].feature_names)))
    with pytest.raises(MC.PlanError, match="REGION_ANNOTATIONS: the transformer applied to it needs a vector Number"):
        MC.compile_plan(VcfHeader("\n".join(hdr) + "\n"), tr, util.fit_model("lr", x, [0, 1, 0, 1]), fl["customs"])


def test_every_reducer_and_policy_is_aimed_at():
    aimed = {c.target[1].split(" ")[0] for c in FC.CASES}
    assert set(FC.REDUCERS) <= aimed | {"RED_LEN"} and {"RED_FIX_QUAL", "RED_FIX_ALLELE0", "RED_FIX_ALLELE1", "RED_FIX_INDEL"} <= aimed
    assert {"POL_VALUE", "POL_ERROR", "POL_NULL", "combine"} <= aimed
    assert {c.flavour for c in FC.CASES} == set(FC.FLAVOURS)
