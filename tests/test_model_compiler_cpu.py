"""CPU: lowering of fitted transformers / models to the plan blob."""
import struct

import numpy as np
import pytest

from tests import util
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader


@pytest.fixture(scope="module")
def ds():
    d = util.make_dataset(n_records=1200, n_custom=5)
    d["df"], d["tr"], d["x"] = util.fit_transformer(d)
    return d


@pytest.mark.parametrize("kind,model_kind", [("lr", MC.MODEL_LOGISTIC), ("gb_small", MC.MODEL_GB_SKLEARN),
                                             ("rf", MC.MODEL_RF_SKLEARN)])
def test_plan_layout(ds, kind, model_kind):
    model = util.fit_model(kind, ds["x"], ds["labels"])
    plan = MC.compile_plan(VcfHeader(ds["header_text"]), ds["tr"], model, ds["customs"])
    hdr = struct.unpack_from("<15I2H4d", plan.blob, 0)
    assert hdr[0] == MC.PLAN_MAGIC and hdr[1] == MC.PLAN_VERSION
    assert hdr[4] == plan.n_features == ds["x"].shape[1] == 46
    assert hdr[7] == model_kind and hdr[8] == 2
    assert len(plan.blob) % 8 == 0
    # stock single_sample layout of SURVEY.md appendix A
    assert plan.feature_names[:7] == ["ad_0", "ad_1", "gt", "gq", "pl_0", "pl_1", "pl_2"]
    assert plan.feature_names[21] == "qual" and plan.feature_names[41:] == ["lcr", "map_unique", "long_hmer",
                                                                             "ug_hcr", "exome"]


def test_threshold_floor_preserves_le_on_float32():
    rng = np.random.default_rng(0)
    t = rng.normal(size=20000) * 10.0 ** rng.integers(-3, 4, size=20000)
    f = MC._f32_floor(t)
    assert np.all(f.astype(np.float64) <= t)
    up = np.nextafter(f, np.float32(np.inf))
    assert np.all(up.astype(np.float64) > t)
    x = rng.normal(size=20000).astype(np.float32) * 10
    assert np.array_equal(x.astype(np.float64) <= t, x <= f)


def test_missing_header_tag_is_a_plan_error(ds):
    model = util.fit_model("lr", ds["x"], ds["labels"])
    hdr = "\n".join(l for l in ds["header"] if "ID=X_GCC" not in l) + "\n"
    with pytest.raises(MC.PlanError, match="x_gcc"):
        MC.compile_plan(VcfHeader(hdr), ds["tr"], model, ds["customs"])


def test_wrong_feature_count_is_a_plan_error(ds):
    from sklearn.linear_model import LogisticRegression

    model = LogisticRegression(max_iter=50).fit(ds["x"][:, :10], ds["labels"])
    with pytest.raises(MC.PlanError, match="features"):
        MC.compile_plan(VcfHeader(ds["header_text"]), ds["tr"], model, ds["customs"])


def test_unfitted_transformer_rejected(ds):
    from variantcalling_b200 import transformers as T
    from variantcalling_b200.tprep_constants import VcfType

    with pytest.raises(MC.PlanError, match="not fitted"):
        MC.compile_plan(VcfHeader(ds["header_text"]), T.get_transformer(VcfType.SINGLE_SAMPLE), None)


def test_xgboost_json_lowering():
    """A hand-written xgboost JSON dump (2 stumps, binary:logistic) lowers to MODEL_XGB."""
    def tree(feat, cond, lv, rv):
        return {"left_children": [1, -1, -1], "right_children": [2, -1, -1], "split_indices": [feat, 0, 0],
                "split_conditions": [cond, lv, rv], "default_left": [0, 0, 0], "base_weights": [0, lv, rv]}
    doc = {"learner": {"objective": {"name": "binary:logistic"},
                       "learner_model_param": {"base_score": "5E-1", "num_class": "0", "num_feature": "3"},
                       "gradient_booster": {"name": "gbtree", "model": {"trees": [tree(0, 0.5, -0.1, 0.2),
                                                                                   tree(2, 1.5, 0.3, -0.4)],
                                                                        "tree_info": [0, 0]}}}}
    m = MC._lower_xgboost_json(doc, 3)
    assert m["kind"] == MC.MODEL_XGB and m["cmp"] == MC.CMP_LT and m["n_trees"] == 2 and m["n_nodes"] == 6
    assert m["init"][0] == 0.0 and m["n_outputs"] == 1 and m["n_classes"] == 2


def test_no_model_plan():
    p = MC.compile_plan_no_model("##fileformat=VCFv4.2\n#CHROM\tPOS\n")
    assert p.n_features == 0 and len(p.blob) == 96


@pytest.mark.parametrize("vtype,extra_info", [("deep_variant", ["VAF"]), ("joint_callset", []),
                                              ("deep_variant_extended", ["MQ0_REF", "MQ0_ALT", "LS_REF"])])
def test_other_vcf_flavours_lower_or_fail_loudly(ds, vtype, extra_info):
    """The DeepVariant / joint feature lists (transformers.py:241-265,289-290) lower through the
    same entries; a flavour whose tags the header lacks is a PlanError, never a silent zero."""
    from sklearn.linear_model import LogisticRegression

    from variantcalling_b200 import transformers as T
    from variantcalling_b200.tprep_constants import VcfType

    tr = T.get_transformer(VcfType(vtype), None)
    names = [e[0] for e in tr.transformers]
    assert names[:4] == ["ad", "gt", "gq", "pl"]
    hdr = ds["header_text"]
    if vtype == "deep_variant":
        hdr = hdr.replace("##FORMAT=<ID=PL", '##FORMAT=<ID=VAF,Number=A,Type=Float,Description="v">\n##FORMAT=<ID=PL')
        df = ds["df"].copy()
        df["vaf"] = [(0.5,)] * len(df)
        import pandas as pd
        with pd.option_context("future.infer_string", False):
            x = tr.fit_transform(df)
        model = LogisticRegression(max_iter=20).fit(x.to_numpy(dtype=float), ds["labels"])
        plan = MC.compile_plan(VcfHeader(hdr), tr, model, None)
        assert plan.feature_names[-1] == "vaf" and plan.n_features == 22
    elif vtype == "joint_callset":
        import pandas as pd
        with pd.option_context("future.infer_string", False):
            x = tr.fit_transform(ds["df"])
        model = LogisticRegression(max_iter=20).fit(x.to_numpy(dtype=float), ds["labels"])
        plan = MC.compile_plan(VcfHeader(hdr), tr, model, None)
        assert plan.n_features == 21 and plan.feature_names[-1] == "x_gcc"
    else:
        # the synthetic header has no MQ0_REF ... tags: lowering must refuse, not guess
        tr.transformers_ = [(n, t, c) for (n, t, c) in tr.transformers]
        with pytest.raises(MC.PlanError):
            MC.compile_plan(VcfHeader(hdr), tr, None, None)


def test_real_deepvariant_header_of_the_reference_compiles():
    """The one real (non-LFS) VCF header in the reference tree, a UG DeepVariant call set with 3366
    contigs (stored as tests/golden/dv_header.txt.gz): the header model reads it, the loader whitelist
    picks its tags, and the ``deep_variant`` flavour fitted on records of that schema lowers against it."""
    import gzip
    import os

    import numpy as np
    import pandas as pd

    from oracle import ref_pipeline as R
    from oracle.vcf_reader import OracleVariantFile
    from tests import dv_data, util
    from variantcalling_b200 import transformers as T
    from variantcalling_b200.tprep_constants import VcfType

    path = os.path.join(os.path.dirname(__file__), "golden", "dv_header.txt.gz")
    with gzip.open(path, "rt") as fh:
        hdr = VcfHeader(fh.read())
    assert len(hdr.contigs) > 3000 and hdr.contigs["chr1"] == 248956422 and hdr.samples
    cols = hdr.loader_columns(dv_data.CUSTOMS)
    assert {"ad", "gt", "gq", "pl", "dp", "vaf", "sor", "af", "x_css", "x_gcc", "x_hil", "x_hin", "x_ic", "x_il", "x_lm", "x_rm",
            "variant_type", "lcr", "ug_hcr"} <= set(cols)
    ds = dv_data.generate(1500, seed=5)
    df = R.get_vcf_df(OracleVariantFile(ds["header_text"].encode() + ds["text"]), None, ds["customs"])
    tr = T.get_transformer(VcfType.DEEP_VARIANT, [c.lower() for c in ds["customs"]])
    with pd.option_context("future.infer_string", False):
        x = tr.fit_transform(R.harness_float_columns(df)).to_numpy(dtype=np.float64)
    plan = MC.compile_plan(hdr, tr, util.fit_model("lr", x, ds["labels"]), ds["customs"])
    ours = MC.compile_plan(VcfHeader(ds["header_text"]), tr, util.fit_model("lr", x, ds["labels"]), ds["customs"])
    assert plan.feature_names == ours.feature_names and plan.tags == ours.tags
