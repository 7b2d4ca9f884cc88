"""GPU: xgboost models with default-left and categorical nodes in K3, bit for bit against the restated predictor
(tests/xgb_categorical_ref.py): the reference's three xgboost models (two srsnv fold models, depth 10 with categorical
splits: k3_infer; the featuremap model, depth 5 with default-left nodes: k3_heap) on seeded frames, generated documents
landing on each K3 kernel and staging, NaN / +-inf at the C ABI, and the srsnv k-fold / ML_QUAL step against the
reference's own output (tests/golden/srsnv_kfold.npz)."""
import os

import numpy as np
import pytest

from tests import xgb_categorical_ref as XR
from variantcalling_b200 import lib
from variantcalling_b200 import model_apply as MA
from variantcalling_b200 import model_compiler as MC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRSNV = [f"416119_L7402.test.model_fold_{k}.json" for k in (0, 1)]
FEATUREMAP = "HG006_HG003.v1.25.WG.t_alt_readsGT1.V1.15.json"


def _split_values(doc) -> dict:
    """feature -> every numeric split condition and the floats one ulp either side of it."""
    out = {}
    for tr in doc["learner"]["gradient_booster"]["model"]["trees"]:
        st = tr.get("split_type") or [0] * len(tr["left_children"])
        for lc, f, c, t in zip(tr["left_children"], tr["split_indices"], tr["split_conditions"], st):
            if lc != -1 and t == 0:
                c = np.float32(c)
                out.setdefault(f, []).extend([c, np.nextafter(c, np.float32(-np.inf)), np.nextafter(c, np.float32(np.inf))])
    return {f: np.unique(np.asarray(v, dtype=np.float32)) for f, v in out.items()}


def _edge_matrix(doc, n_features, n, seed, cat_codes=None):
    """Rows: every numeric feature at one of its split values +-1 ulp (each value used), 8% NaN; categorical
    features (cat_codes: feature -> number of codes) at a code, an unknown one (NaN), a negative or too large one."""
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 50, size=(n, n_features)).astype(np.float32)
    for f, vals in _split_values(doc).items():
        x[:, f] = vals[np.arange(n) % vals.size][rng.permutation(n)] if vals.size <= n else rng.choice(vals, n)
    for f, k in (cat_codes or {}).items():
        x[:, f] = rng.choice(np.array([*range(k), np.nan, -1.0, 2.5, 40.0, 1024.0, 2.0 ** 24], dtype=np.float32), n,
                             p=[0.85 / k] * k + [0.05, 0.02, 0.02, 0.02, 0.02, 0.02])
    x[rng.random(x.shape) < 0.08] = np.nan
    return x


def _run(doc, x):
    clf = MA.GpuClassifier(doc, n_features=x.shape[1], max_rows=max(1, x.shape[0]))
    try:
        return clf.predict_proba(x), clf.ctx.k3_config()
    finally:
        clf.close()


@pytest.mark.parametrize("name", SRSNV)
def test_srsnv_fold_models_bit_for_bit(name):
    """The reference's srsnv fold model on a frame built from its category value maps: categoricals with unknown
    values, numerics at every split value +-1 ulp and NaN."""
    doc = XR.load_golden_json(name)
    features = XR.metadata_features()
    names = [f["name"] for f in features]
    n = 6000
    raw = XR.srsnv_frame(31, n, features)
    edges = _split_values(doc)
    rng = np.random.default_rng(5)
    for i, f in enumerate(features):
        if f["type"] != "c" and i in edges:
            v = edges[i][rng.integers(0, edges[i].size, n)].astype(np.float64)
            v[rng.random(n) < 0.08] = np.nan
            raw[f["name"]] = v
    df = MA.set_categorical_columns(raw, {f["name"]: list(f["values"]) for f in features if f["type"] == "c"})[names]
    got, cfg = _run(doc, df)
    want = XR.predict_proba(doc, MA.frame_matrix(df, names)).astype(np.float64)
    assert cfg["walk"] == "categorical" and cfg["kernel"] == "infer"
    assert np.array_equal(got, want)
    with pytest.raises(ValueError, match="feature_names mismatch"):
        _run(doc, df[names[::-1]])


def test_featuremap_model_bit_for_bit():
    doc = XR.load_golden_json(FEATUREMAP)
    n_features = int(doc["learner"]["learner_model_param"]["num_feature"])
    x = _edge_matrix(doc, n_features, 8000, 3)
    got, cfg = _run(doc, x)
    assert cfg["walk"] == "categorical" and cfg["kernel"] == "heap" and cfg["resident"]
    assert np.array_equal(got, XR.predict_proba(doc, x).astype(np.float64))


# generated documents: (n_features, trees, depth, full depth, leaf_p) -> expected (kernel, resident)
GENERATED = {
    "heap_resident": ((30, 60, 6, False, 0.3), ("heap", True)),
    "heap_chunked": ((40, 200, 8, True, 0.0), ("heap", False)),
    "infer_resident": ((26, 200, 10, False, 0.3), ("infer", True)),
    "infer_chunked": ((26, 120, 12, False, 0.15), ("infer", False)),
}


@pytest.mark.parametrize("case", sorted(GENERATED))
def test_generated_categorical_documents_on_every_staging(case):
    (f, n_trees, depth, full, leaf_p), (kernel, resident) = GENERATED[case]
    wide_p = 0.1 if resident else 0.0  # long bitsets in the resident cases; the chunked forests are large enough
    cat_features = range(0, f, 3)
    rng = np.random.default_rng(len(case))
    base = rng.normal(0, 1, size=(400, f)).astype(np.float32)
    base[:, list(cat_features)] = rng.integers(0, 14, size=(400, len(cat_features)))
    doc = XR.categorical_document(17 + len(case), base, n_trees, cat_features, max_depth=depth, full_depth=full,
                                  leaf_p=leaf_p, num_class=2 if "infer" in case else 0, wide_p=wide_p)
    x = _edge_matrix(doc, f, 3000, 11, cat_codes={c: 14 for c in cat_features})
    got, cfg = _run(doc, x)
    assert (cfg["kernel"], cfg["resident"], cfg["walk"]) == (kernel, resident, "categorical"), cfg
    assert np.array_equal(got, XR.predict_proba(doc, x).astype(np.float64))


def test_plain_plans_keep_the_plain_walk_and_inf_is_refused(gpu_ctx):
    from oracle import xgb_predictor as XP
    from sklearn.ensemble import GradientBoostingClassifier

    rng = np.random.default_rng(2)
    x = rng.normal(size=(500, 6)).astype(np.float32)
    plain = XP.random_gbtree_document(3, x, 20, max_depth=5)
    sk = GradientBoostingClassifier(n_estimators=5, max_depth=3).fit(x.astype(np.float64), x[:, 0] > 0)
    for model in (plain, sk):
        gpu_ctx.load_plan(MC.compile_plan_model_only(model, 6).blob)
        gpu_ctx.reserve(4096, 1024, 1)
        assert gpu_ctx.k3_config()["walk"] == "plain"
    # a plain xgboost plan takes NaN (every default child is the right one: the plain walk's NaN route)
    gpu_ctx.load_plan(MC.compile_plan_model_only(plain, 6).blob)
    gpu_ctx.reserve(4096, 1024, 1)
    gpu_ctx.enable_phreds(2)
    gpu_ctx.reserve(4096, 1024, 1)
    xn = x.copy()
    xn[rng.random(xn.shape) < 0.2] = np.nan
    gpu_ctx.predict_features(xn)
    assert np.array_equal(gpu_ctx.collect_phreds(0, 500), XR.predict_proba(plain, xn).astype(np.float64))
    for v in (np.inf, -np.inf):
        bad = x.copy()
        bad[7, 4] = v
        with pytest.raises(lib.UgvcDataError):
            gpu_ctx.predict_features(bad)
        assert gpu_ctx.last_data_error()[:2] == (7, 4)
    gpu_ctx.load_plan(MC.compile_plan_model_only(sk, 6).blob)  # sklearn: NaN is still refused
    gpu_ctx.reserve(4096, 1024, 1)
    with pytest.raises(lib.UgvcDataError):
        gpu_ctx.predict_features(xn)


def _reordered(doc, names):
    """The same model with its features in another column order (feature_names / feature_types / split_indices)."""
    import copy

    doc = copy.deepcopy(doc)
    learner = doc["learner"]
    old = learner["feature_names"]
    perm = [names.index(nm) for nm in old]  # old index -> new index
    learner["feature_types"] = [learner["feature_types"][old.index(nm)] for nm in names]
    learner["feature_names"] = list(names)
    for tr in learner["gradient_booster"]["model"]["trees"]:
        tr["split_indices"] = [perm[i] for i in tr["split_indices"]]
    return doc


def test_k_fold_and_ml_qual_against_the_reference_golden():
    g = np.load(os.path.join(ROOT, "tests", "golden", "srsnv_kfold.npz"))
    features = XR.metadata_features()
    names = [f["name"] for f in features]
    cat_dict = {f["name"]: list(f["values"]) for f in features if f["type"] == "c"}
    n = g["x"].shape[0]
    raw = XR.srsnv_frame(2024, n, features)
    df = MA.set_categorical_columns(raw, cat_dict)
    df["fold_id"] = XR.srsnv_folds(7, n)
    docs = [XR.load_golden_json(nm) for nm in SRSNV]
    models = [MA.GpuClassifier(d, n_features=len(names), max_rows=n) for d in docs]
    try:
        got = MA.k_fold_predict_proba(models, df, names, 2)
        assert np.array_equal(got.to_numpy(), g["preds"], equal_nan=True)
    finally:
        for m in models:
            m.close()
    # ML_QUAL: folds by chromosome; the models in the srsnv order (numerical features, then categorical ones)
    numerical = [f["name"] for f in features if f["type"] != "c"]
    ordered = [_reordered(d, numerical + list(cat_dict)) for d in docs]
    chrom_of = {0.0: "chr1", 1.0: "chr2", -1.0: "chrM", 2.0: "chr3", 5.0: "chr5"}
    raw["chrom"] = [chrom_of.get(v, "chrX") for v in g["fold"]]
    models = [MA.GpuClassifier(d, n_features=len(names), max_rows=n) for d in ordered]
    try:
        q = MA.ml_qual(models, raw, cat_dict, numerical, chrom_folds={"chr1": 0, "chr2": 1, "chrM": -1, "chr3": 2, "chr5": 5})
    finally:
        for m in models:
            m.close()
    with np.errstate(divide="ignore"):
        want = (-10 * np.log10(1 - g["preds"])).clip(min=0)
    assert np.array_equal(q, want, equal_nan=True)
