"""GPU: the documented deviations of DESIGN.md section 4, pinned as tests -- each one either reproduces what the
reference does or asserts the stated difference, so that none of them can drift silently.

 1. an optional numeric tag missing from EVERY record of a contig: the reference's pandas frame holds an all-None
    object column that SimpleImputer does not impute and _validate_data then asserts (variant_filtering_utils.py:
    128-143); the plan applies the imputer's constant per record, so the device returns the scores the reference
    gives as soon as one record of the contig carries the tag.
 2. integer tag values beyond 2^24 with a logistic-regression model: sklearn evaluates the frame in fp64, the
    feature matrix on the device is fp32 (X.astype(float32), what the tree models see in the reference too): the
    probability may differ, by no more than the coefficient times the fp32 rounding of the value.
 3. an Integer literal outside int32: htslib refuses it, the oracle reader (Python int) keeps it; the device refuses
    the record (UgvcDataError naming it).
 4. an empty numeric value ("SOR=", "LONG_HMER="): the reference reads None and imputes it; the device refuses the
    record as a bad literal.
 5. an empty string value where the reference indexes or iterates it ("X_HIN=" is (), "X_LM=" under Number=1 is None):
    the reference raises, the device scores a string without a base (0).
The cases of 3-5 are in tests/feature_cases.py (``deviation``); the reference side is pinned by
tests/test_feature_cases_cpu.py.
"""
import numpy as np
import pandas as pd
import pytest

from oracle import ref_pipeline as R
from oracle.vcf_reader import OracleVariantFile
from tests import util
from variantcalling_b200 import lib
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def base():
    ds = util.make_dataset(n_records=1500, n_custom=2, seed=404)
    _, tr, x = util.fit_transformer(ds)
    return ds, tr, x


def drop_tag(line: str, tag: str) -> str:
    cols = line.split("\t")
    cols[7] = ";".join(kv for kv in cols[7].split(";") if not kv.startswith(tag + "="))
    return "\t".join(cols)


def test_all_none_optional_column(gpu_ctx, base):
    ds, tr, x = base
    model = util.fit_model("gb_small", x, ds["labels"])
    chr1 = [ln for ln in ds["lines"] if ln.startswith("chr1\t")]
    assert len(chr1) > 60
    lines = [drop_tag(ln, "SOR") for ln in chr1[:-1]]  # SOR: an imputed (NaN -> 0) float of the stock list
    text = ("\n".join(lines) + "\n").encode()
    header_text = ds["header_text"]
    # the reference path on exactly these records: an all-None column reaches _validate_data
    vf = OracleVariantFile(header_text.encode() + text)
    with pytest.raises((AssertionError, ValueError, TypeError)):
        R.filter_variants(vf, model, tr, custom_annotations=ds["customs"])
    # ... and with one more record that has the tag it scores them: the device gives those scores without the extra record
    extra = chr1[-1]  # same contig: the reference builds one frame per contig
    assert "SOR=" in extra
    vf2 = OracleVariantFile(header_text.encode() + text + (extra + "\n").encode())
    exp = R.filter_variants(vf2, model, tr, custom_annotations=ds["customs"])
    plan = MC.compile_plan(VcfHeader(header_text), tr, model, ds["customs"])
    gpu_ctx.load_plan(plan.blob)
    gpu_ctx.set_key_order(*lib.learn_key_order(text))
    gpu_ctx.reserve(len(text) + 4096, len(lines) + 16, 1)
    res = gpu_ctx.filter_batch(text, 30.0)
    assert res["n_records"] == len(lines)
    np.testing.assert_allclose(res["probs"], exp["probs"][: len(lines)], atol=1e-5, rtol=0)
    low = np.array(["LOW_SCORE" in f.split(";") for f in exp["filters"][: len(lines)]])
    assert np.array_equal(res["low_score"].astype(bool), low)


def test_large_integers_under_logistic_regression(gpu_ctx, base):
    ds, tr, x = base
    model = util.fit_model("lr", x, ds["labels"])
    big = 16_777_217  # 2^24 + 1: not a float32
    lines = list(ds["lines"][:200])
    cols = lines[5].split("\t")
    cols[7] = ";".join(("AN=%d" % big) if kv.startswith("AN=") else kv for kv in cols[7].split(";"))
    lines[5] = "\t".join(cols)
    text = ("\n".join(lines) + "\n").encode()
    vf = OracleVariantFile(ds["header_text"].encode() + text)
    exp = R.filter_variants(vf, model, tr, custom_annotations=ds["customs"])
    plan = MC.compile_plan(VcfHeader(ds["header_text"]), tr, model, ds["customs"])
    gpu_ctx.load_plan(plan.blob)
    gpu_ctx.set_key_order(*lib.learn_key_order(text))
    gpu_ctx.reserve(len(text) + 4096, len(lines) + 16, 1)
    res = gpu_ctx.filter_batch(text, 30.0)
    feats = gpu_ctx.debug_features(res["n_records"]).T
    df = R.harness_float_columns(R.get_vcf_df(vf, None, ds["customs"]))
    with pd.option_context("future.infer_string", False):
        want64 = tr.transform(df).to_numpy(dtype=np.float64)
    assert np.array_equal(feats, want64.astype(np.float32))            # the matrix is the reference's, cast to fp32
    col = int(np.flatnonzero(want64[5] == big)[0])
    assert feats[5, col] == np.float32(big) and float(np.float32(big)) != float(big)  # ... where 2^24 + 1 is not representable
    # every other record agrees to 1e-9; record 5 differs by at most |coef| * |rounding| in the margin
    others = np.ones(len(lines), dtype=bool)
    others[5] = False
    np.testing.assert_allclose(res["probs"][others], exp["probs"][others], atol=1e-6, rtol=0)
    margin_err = abs(float(model.coef_[0][col])) * abs(float(np.float32(big)) - big)
    assert abs(float(res["probs"][5, 1]) - float(exp["probs"][5, 1])) <= margin_err * 0.25 + 1e-6  # d sigmoid <= 1/4


@pytest.mark.parametrize("name", ["ss", "ss1", "dvx", "cnv"])
def test_corpus_deviations(gpu_ctx, name):
    from tests import feature_cases as FC
    from tests.test_gpu_feature_edges import fitted, plan_of, run

    fl, tr, _ = fitted(name)
    plan = plan_of(name, "gb8")
    clean = fl["lines"][:40]
    learn = ("\n".join(fl["lines"][:120]) + "\n").encode()
    cases = [c for c in FC.cases_of(name) if c.deviation]
    assert cases
    for c in cases:
        line = FC.apply(FC.base_record(fl), c.edits)
        if c.want == FC.RAISES:
            with pytest.raises((ValueError, KeyError, AssertionError, TypeError, IndexError)):
                FC.reference_matrix(fl, clean + [line], tr)
        else:
            FC.reference_matrix(fl, clean + [line], tr)
        for legacy in (False, True):
            res = run(gpu_ctx, plan.blob, clean + [line], learn, legacy)
            if c.on_device == FC.RAISES:
                assert res.get("error", (None,))[0] == len(clean), (c.name, legacy)
                continue
            assert "error" not in res, (c.name, legacy, res.get("error"))
            for feat, v in c.on_device.items():
                got = res["feats"][len(clean), plan.feature_names.index(feat)]
                assert got.tobytes() == np.float32(v).tobytes(), (c.name, feat, got)
