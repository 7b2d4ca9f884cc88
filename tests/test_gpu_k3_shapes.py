"""GPU: K3 in every launch configuration it has, against the estimators themselves.

The K3 launch depends on the model (kernels.cu: k3_choose, k3h_shape, k3h_chunk_trees, k3_tpb,
k3_chunk_nodes): k3_heap in one of nine template shapes with the forest resident or staged in chunks of trees,
or k3_infer (forests deeper than 8 or with >= 65536 leaf rows) with the forest resident or staged in chunks of
nodes.  Every case below is sized to land on one configuration and asserts it through ugvc_test_k3_config, then
compares the device with sklearn's own predict_proba on the fp32 matrix (GB / RF <= 1e-12, LR <= 1e-9) or with
the xgboost restatement bit for bit, at rows sitting on the split thresholds, special values and row counts
around the tile and the persistent wave."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import ref_pipeline as R
from oracle import xgb_predictor as XP
from tests import util
from variantcalling_b200 import lib
from variantcalling_b200 import model_compiler as MC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N_BASE = 1500   # rows the oracles score; longer runs repeat them
SPECIALS = np.array([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -3e-39, 1e30, -1e30], dtype=np.float32)


def _train(seed, n, f, k):
    """A random matrix and labels that depend on a few columns plus noise (k classes)."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, f)).astype(np.float32).astype(np.float64)
    x[:, ::7] = np.round(x[:, ::7] * 3)  # a few integer-valued columns: ties and repeated thresholds
    s = x[:, 0] - 0.7 * x[:, 1 % f] + 0.5 * x[:, 2 % f] * x[:, 3 % f] + rng.normal(0, 1.0, n)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, k + 1)[1:-1]))
    return x, y


def _sk(kind, k, f, seed=5, n=600, **kw):
    from sklearn.ensemble import GradientBoostingClassifier, RandomForestClassifier
    from sklearn.linear_model import LogisticRegression

    x, y = _train(seed, n, f, k)
    if kind == "lr":
        m = LogisticRegression(max_iter=500)
    elif kind == "gb":
        m = GradientBoostingClassifier(learning_rate=0.2, subsample=0.5, max_features=0.3, random_state=0, **kw)
    else:
        m = RandomForestClassifier(random_state=0, n_jobs=1, **kw)
    return m.fit(x, y)


def _rf_many_leaves():
    """A depth-8 RF with 65536 leaf rows or more: 800 trees on striped 3-class labels (~90 leaves a tree)."""
    from sklearn.ensemble import RandomForestClassifier

    x, _ = _train(9, 3000, 20, 3)
    y = (np.floor((x[:, 0] + x[:, 1] + x[:, 2]) * 40) % 3).astype(int)
    return RandomForestClassifier(n_estimators=800, max_depth=8, random_state=0, n_jobs=1).fit(x, y)


def _xgb(f, n_trees, num_class=0, seed=11, **kw):
    x = _base(seed, f)
    return XP.random_gbtree_document(seed, x[:400], n_trees, num_class=num_class, **kw)


def _base(seed, f):
    """N_BASE rows: ordinary values with a sprinkle of +-0, subnormals and +-1e30, plus rows made only of them."""
    rng = np.random.default_rng(seed + 1000)
    x = rng.normal(size=(N_BASE, f)).astype(np.float32)
    x[:, ::7] = np.round(x[:, ::7] * 3)
    hit = rng.random(x.shape) < 0.02
    x[hit] = rng.choice(SPECIALS, size=int(hit.sum()))
    for i, v in enumerate(SPECIALS):
        x[i] = v
    return x


def _sk_thresholds(model):
    """feature -> fp64 split thresholds of every tree of a fitted sklearn forest."""
    out = {}
    for e in np.ravel(model.estimators_):
        t = e.tree_
        for f, thr in zip(t.feature, t.threshold):
            if f >= 0:
                out.setdefault(int(f), []).append(float(thr))
    return out


def _edge_rows(x, model, rng, n=300):
    """Rows whose every split feature sits on a threshold's decision boundary: for sklearn the fp32 floor of a
    threshold and the next float up, for xgboost the split condition and the float below it."""
    if isinstance(model, dict):
        cand = {}
        for tr in model["learner"]["gradient_booster"]["model"]["trees"]:
            for lc, f, c in zip(tr["left_children"], tr["split_indices"], tr["split_conditions"]):
                if lc != -1:
                    c = np.float32(c)
                    cand.setdefault(f, []).extend([c, np.nextafter(c, np.float32(-np.inf))])
    elif hasattr(model, "estimators_"):
        cand = {}
        for f, ts in _sk_thresholds(model).items():
            lo = MC._f32_floor(np.asarray(ts))  # noqa: SLF001
            cand[f] = list(lo) + list(np.nextafter(lo, np.float32(np.inf)))
    else:
        return x[:0]
    rows = x[rng.integers(0, x.shape[0], n)].copy()
    for f, vals in cand.items():
        vals = np.asarray(vals, dtype=np.float32)
        rows[:, f] = vals[rng.integers(0, vals.size, n)]
    return rows


def _forest_size(model):
    """(trees, preorder nodes) of a forest; (0, 0) for a linear model."""
    if isinstance(model, dict):
        trees = model["learner"]["gradient_booster"]["model"]["trees"]
        return len(trees), sum(len(t["left_children"]) for t in trees)
    if not hasattr(model, "estimators_"):
        return 0, 0
    est = np.ravel(model.estimators_)
    return len(est), sum(e.tree_.node_count for e in est)


def _oracle(model, x32):
    if isinstance(model, dict):
        return XP.predict_proba(model, x32).astype(np.float64)
    if type(model).__name__ == "LogisticRegression":
        return model.predict_proba(x32.astype(np.float64))
    return model.predict_proba(x32)


# name -> (model builder, n_features, expected configuration).  Shapes of k3_heap (kernels.cu: k3h_tile_bytes =
# nbuf * F * tpb * 4 + 12 F + 64 B, a depth-d tree takes 10 * 2^d B, 224 KiB in all): resident in the first shape
# whose tile + forest fits; else chunks of 16 k depth-8 trees in the first of 256x2 (F <= 91), 192x2 (<= 121),
# 128x2 (<= 181), 128x1 that fits tile + 16 trees.
HEAP = "heap"
CASES = {
    "lr2_heap512_res": (lambda: _sk("lr", 2, 46), 46, (HEAP, 512, 1, 2, True)),
    "lr4_heap128x1_res": (lambda: _sk("lr", 4, 250), 250, (HEAP, 128, 1, 1, True)),
    "gb2_heap512_res": (lambda: _sk("gb", 2, 46, n_estimators=12, max_depth=4), 46, (HEAP, 512, 1, 2, True)),
    "gb3_heap448_res": (lambda: _sk("gb", 3, 100, n_estimators=15, max_depth=6), 100, (HEAP, 448, 1, 2, True)),
    "rf3_heap384_res": (lambda: _sk("rf", 3, 120, n_estimators=50, max_depth=6), 120, (HEAP, 384, 1, 2, True)),
    "xgb2_heap128x2_res": (lambda: _xgb(200, 30, max_depth=6, full_depth=True), 200, (HEAP, 128, 2, 1, True)),
    "gb2_250f_heap128x1_res": (lambda: _sk("gb", 2, 250, n_estimators=100, max_depth=6), 250, (HEAP, 128, 1, 1, True)),
    "rf2_300x4_heap512_res": (lambda: _sk("rf", 2, 46, n_estimators=300, max_depth=4), 46, (HEAP, 512, 1, 2, True)),
    "xgbm2_small_res": (lambda: _xgb(46, 40, num_class=2, max_depth=5, tree_info="shuffled"), 46, (HEAP, 512, 1, 2, True)),
    "xgbm3_heap256x2_chunk": (lambda: _xgb(46, 150, num_class=3, max_depth=8, full_depth=True), 46, (HEAP, 256, 2, 1, False)),
    "gb4_heap256x2_chunk": (lambda: _sk("gb", 4, 46, n_estimators=25, max_depth=8), 46, (HEAP, 256, 2, 1, False)),
    "rf2_heap192x2_chunk": (lambda: _sk("rf", 2, 100, n_estimators=80, max_depth=8), 100, (HEAP, 192, 2, 1, False)),
    "xgb2_heap192x2_chunk": (lambda: _xgb(100, 80, max_depth=8, full_depth=True), 100, (HEAP, 192, 2, 1, False)),
    "gb2_heap128x2_chunk": (lambda: _sk("gb", 2, 150, n_estimators=70, max_depth=8), 150, (HEAP, 128, 2, 1, False)),
    "xgbm4_heap128x1_chunk": (lambda: _xgb(200, 100, num_class=4, max_depth=8, full_depth=True, tree_info="blocks"), 200,
                              (HEAP, 128, 1, 1, False)),
    "xgbm3_infer_res": (lambda: _xgb(20, 30, num_class=3, max_depth=12, tree_info="shuffled"), 20, ("infer", 384, 1, 1, True)),
    "rf2_deep_infer_res": (lambda: _sk("rf", 2, 20, n_estimators=10), 20, ("infer", 384, 1, 1, True)),
    "xgbm2_srsnv_200x10_infer_chunk": (lambda: _xgb(46, 400, num_class=2, max_depth=10, full_depth=True, leaf_p=0.15), 46,
                                       ("infer", 256, 1, 1, False)),
    "rf3_800x8_leafrows_infer_chunk": (_rf_many_leaves, 20, ("infer", 256, 1, 1, False)),
}
_MODELS: dict = {}


def _model(name):
    if name not in _MODELS:
        _MODELS[name] = CASES[name][0]()
    return _MODELS[name]


@pytest.fixture(scope="module")
def ctx():
    c = lib.Context(0)
    c.enable_phreds(2)  # the fp64 class probabilities next to the fp32 ones
    yield c
    c.close()


def _load(ctx, model, f, rows):
    ctx.load_plan(MC.compile_plan_model_only(model, f).blob)
    ctx.reserve(4096, max(rows, 1), 1)
    return ctx.k3_config()


def _predict(ctx, x, thr):
    ctx.counts_reset()
    res = ctx.predict_features(x, threshold=thr)
    res["p64"] = ctx.collect_phreds(0, x.shape[0])
    res["counts"] = ctx.counts()
    return res


def _same(a, b, n):
    """Device results of one row set agree bit for bit on its first n rows."""
    for k in ("low_score", "probs", "qual", "p64"):
        assert np.array_equal(a[k][:n].view(np.uint8), b[k][:n].view(np.uint8)), k


def _check_against_oracle(res, model, x, thr):
    want = _oracle(model, x)
    got = res["p64"][: x.shape[0]]
    assert got.shape == want.shape
    if isinstance(model, dict):  # xgboost: fp32 margins and link, bit for bit
        assert np.array_equal(got, want), np.argwhere(got != want)[:5]
        assert np.array_equal(res["probs"][: x.shape[0]], want.astype(np.float32))
    else:
        tol = 1e-9 if type(model).__name__ == "LogisticRegression" else 1e-12
        np.testing.assert_allclose(got, want, atol=tol, rtol=0)
    _, q, _ = R.score_math(want)
    np.testing.assert_allclose(res["qual"][: x.shape[0]], q, atol=1e-6, rtol=1e-12)
    low = res["low_score"][: x.shape[0]].astype(bool)
    assert np.array_equal(low, res["qual"][: x.shape[0]] <= thr)
    clear = np.abs(q - thr) > 1e-6
    assert np.array_equal(low[clear], (q <= thr)[clear])
    return want.size


@pytest.mark.parametrize("name", list(CASES))
def test_k3_configuration_against_the_estimator(ctx, name):
    _, f, (kernel, tpb, nbuf, groups, resident) = CASES[name]
    model = _model(name)
    rng = np.random.default_rng(len(name))
    base = _base(7, f)
    x = np.concatenate([_edge_rows(base, model, rng), base])[:N_BASE]
    cfg = _load(ctx, model, f, 1)
    assert (cfg["kernel"], cfg["tpb"], cfg["nbuf"], cfg["groups"], cfg["resident"]) == (kernel, tpb, nbuf, groups, resident), cfg
    n_trees, n_nodes = _forest_size(model)
    if kernel == HEAP and not resident:  # whole groups of 16 trees per chunk, several chunks
        assert cfg["chunk"] % 16 == 0 and 0 < cfg["chunk"] < n_trees, cfg
    if kernel == "infer" and not resident:
        assert 0 < 3 * cfg["chunk"] < n_nodes, cfg
    if name.startswith("rf3_800x8"):  # a forest of depth <= 8 without a heap form: 65536 leaf rows or more
        assert max(e.get_depth() for e in model.estimators_) <= 8
        assert sum(e.tree_.n_leaves for e in model.estimators_) >= 65536
    # row counts around the tile (gs records) and the persistent wave (grid x groups x gs records)
    gs, wave = cfg["gs"], cfg["grid"] * cfg["groups"] * cfg["gs"]
    n_full = max(N_BASE, wave + 1)
    xf = np.resize(x, (n_full, f))  # repeats the oracle's rows
    ctx.reserve(4096, n_full, 1)
    thr = float(np.quantile(R.score_math(_oracle(model, x[:200]))[1], 0.4)) + 1e-3
    full = _predict(ctx, xf, thr)
    _check_against_oracle(full, model, x, thr)
    rep = np.arange(n_full) % N_BASE  # every repeat of a row scores the same
    for k in ("low_score", "probs", "qual", "p64"):
        assert np.array_equal(full[k], full[k][rep]), k
    low = int(full["low_score"].sum())
    assert full["counts"]["n_records"] == n_full and full["counts"]["n_low_score"] == low
    assert full["counts"]["n_pass"] == n_full - low
    for n in sorted({1, gs - 1, gs, gs + 1, wave - 1, wave, 1000 + 37}):
        part = _predict(ctx, xf[:n], thr)
        _same(part, full, n)
        assert part["counts"]["n_records"] == n and part["counts"]["n_low_score"] == int(part["low_score"].sum())


def test_plans_loaded_in_turn(ctx):
    """chunked -> resident -> chunked on one context: every plan scores as it did alone."""
    names = ["gb2_heap128x2_chunk", "lr2_heap512_res", "xgbm2_srsnv_200x10_infer_chunk", "gb2_heap128x2_chunk",
             "rf2_heap192x2_chunk", "xgbm3_infer_res", "rf2_heap192x2_chunk"]
    first = {}
    for name in names:
        f = CASES[name][1]
        x = _base(3, f)
        _load(ctx, _model(name), f, N_BASE)
        res = _predict(ctx, x, 20.0)
        if name in first:
            _same(res, first[name], N_BASE)
        else:
            _check_against_oracle(res, _model(name), x, 20.0)
            first[name] = res


# ------------------------------------------------------------------------------------------ the VCF entry point
@pytest.fixture(scope="module")
def vcf_ds():
    d = util.make_dataset(n_records=2000, n_custom=4, seed=19)
    d["df"], d["tr"], d["x"] = util.fit_transformer(d)
    return d


@pytest.mark.parametrize("depth,n_trees,kernel,resident", [(8, 200, HEAP, False), (10, 30, "infer", True)])
def test_filter_batch_fused_k2_with_chunked_and_deep_forests(vcf_ds, depth, n_trees, kernel, resident):
    """K2's missing / absent policies run inside k3_heap's tile load (K2 + k3_infer for the deep model)."""
    from sklearn.ensemble import GradientBoostingClassifier

    from variantcalling_b200.vcf_header import VcfHeader

    ds = vcf_ds
    model = GradientBoostingClassifier(n_estimators=n_trees, learning_rate=0.1, subsample=0.4, max_depth=depth,
                                       random_state=0).fit(ds["x"], ds["labels"])
    assert max(e.get_depth() for e in model.estimators_.ravel()) == depth
    c = lib.Context(0)
    try:
        c.load_plan(MC.compile_plan(VcfHeader(ds["header_text"]), ds["tr"], model, ds["customs"]).blob)
        cfg = c.k3_config()
        assert (cfg["kernel"], cfg["resident"]) == (kernel, resident), cfg
        c.enable_phreds(2)
        c.set_key_order(*lib.learn_key_order(ds["text"]))
        c.reserve(len(ds["text"]) + 1024, len(ds["lines"]) + 16, 1)
        res = c.filter_batch(ds["text"], 30.0)
        n = res["n_records"]
        assert n == len(ds["lines"])
        p64 = c.collect_phreds(0, n)
        x32 = ds["x"].astype(np.float32)
        assert np.array_equal(c.debug_features(n).T, x32)
        np.testing.assert_allclose(p64, model.predict_proba(x32), atol=1e-12, rtol=0)
        exp = R.filter_variants(ds["vf"], model, ds["tr"], custom_annotations=ds["customs"], decision_threshold=30.0)
        low = np.array(["LOW_SCORE" in f.split(";") for f in exp["filters"]])
        assert np.array_equal(res["low_score"].astype(bool), low)
    finally:
        c.close()


# ------------------------------------------------------------------------------------------ plan-size boundary
@pytest.mark.parametrize("f", [1, 219, 220, 224, 225, 250])
def test_plans_up_to_250_features_load_and_score(ctx, f):
    rng = np.random.default_rng(f)
    doc = _xgb(f, 20, seed=f, max_depth=8, full_depth=True)
    lr = _sk("lr", 2, f, seed=f)
    for model in (doc, lr):
        cfg = _load(ctx, model, f, N_BASE)
        assert cfg["kernel"] == HEAP
        x = np.concatenate([_edge_rows(_base(f, f), model, rng, 200), _base(f, f)])[:N_BASE]
        _check_against_oracle(_predict(ctx, x, 20.0), model, x, 20.0)


def test_deep_forest_feature_limit(ctx):
    """k3_infer holds a 256-record tile: a deep forest loads up to 219 features and is refused above, by name."""
    doc = _xgb(219, 20, seed=3, max_depth=10, full_depth=True)
    cfg = _load(ctx, doc, 219, N_BASE)
    assert cfg["kernel"] == "infer" and cfg["tpb"] == 256
    x = _base(3, 219)
    _check_against_oracle(_predict(ctx, x, 20.0), doc, x, 20.0)
    doc = _xgb(230, 20, seed=3, max_depth=10, full_depth=True)
    with pytest.raises(lib.UgvcError) as e:
        ctx.load_plan(MC.compile_plan_model_only(doc, 230).blob)
    assert e.value.code == lib.UGVC_E_PLAN and "at most 219 features" in e.value.message and "230" in e.value.message


# ------------------------------------------------------------------------------------------ every compiled shape
_CHILD = r"""
import json, sys
import numpy as np
from variantcalling_b200 import lib
blob, x, out = open(sys.argv[1], "rb").read(), np.load(sys.argv[2]), sys.argv[3]
c = lib.Context(0)
c.enable_phreds(2)
c.load_plan(blob)
c.reserve(4096, x.shape[0], 1)
res = c.predict_features(x, threshold=20.0)
np.savez(out, low=res["low_score"], probs=res["probs"], qual=res["qual"], p64=c.collect_phreds(0, x.shape[0]))
cfg, err = c.k3_config(), ""
if len(sys.argv) > 4:
    try:
        c.load_plan(open(sys.argv[4], "rb").read())
    except lib.UgvcError as e:
        err = e.message
print(json.dumps({"cfg": cfg, "err": err}))
c.close()
"""


def _child(tmp_path, env_extra, blob, x, other_blob=None):
    bp, xp, op = tmp_path / "plan.bin", tmp_path / "x.npy", tmp_path / f"out_{len(os.listdir(tmp_path))}.npz"
    bp.write_bytes(blob)
    np.save(xp, x)
    args = [sys.executable, "-c", _CHILD, str(bp), str(xp), str(op)]
    if other_blob is not None:
        (tmp_path / "other.bin").write_bytes(other_blob)
        args.append(str(tmp_path / "other.bin"))
    env = dict(os.environ, **env_extra)
    r = subprocess.run(args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    info = json.loads(r.stdout.strip().splitlines()[-1])
    return info["cfg"], info["err"], dict(np.load(op))


def test_every_compiled_shape_scores_identically(tmp_path):
    """UGVC_K3_SHAPE 0-7, UGVC_K3_NCH448=12 and UGVC_K3_LEGACY=1 (read once per process: one child each) on one
    model every shape holds resident: outputs bit-identical across all of them."""
    model = _sk("gb", 3, 20, n_estimators=8, max_depth=5)
    blob = MC.compile_plan_model_only(model, 20).blob
    x = np.concatenate([_edge_rows(_base(5, 20), model, np.random.default_rng(5), 300), _base(5, 20)])
    shapes = [(512, 1, 2), (448, 1, 2), (384, 1, 2), (256, 2, 1), (192, 2, 1), (128, 2, 1), (256, 1, 1), (128, 1, 1)]
    runs = []
    for i, sh in enumerate(shapes):
        cfg, _, out = _child(tmp_path, {"UGVC_K3_SHAPE": str(i)}, blob, x)
        assert (cfg["kernel"], cfg["tpb"], cfg["nbuf"], cfg["groups"], cfg["resident"]) == ("heap", *sh, True)
        runs.append(out)
    cfg, _, out = _child(tmp_path, {"UGVC_K3_SHAPE": "1", "UGVC_K3_NCH448": "12"}, blob, x)
    assert (cfg["tpb"], cfg["nch"]) == (448, 12)
    runs.append(out)
    # the legacy kernel on the same model; a plan only k3_heap holds is refused at load time, by name
    wide = MC.compile_plan_model_only(_sk("lr", 2, 250), 250).blob
    cfg, err, out = _child(tmp_path, {"UGVC_K3_LEGACY": "1"}, blob, x, other_blob=wide)
    assert cfg["kernel"] == "infer"
    assert "UGVC_K3_LEGACY" in err and "at most 224 features" in err
    runs.append(out)
    np.testing.assert_allclose(runs[0]["p64"], model.predict_proba(x), atol=1e-12, rtol=0)
    for r in runs[1:]:
        for k in ("low", "probs", "qual", "p64"):
            assert np.array_equal(r[k].view(np.uint8), runs[0][k].view(np.uint8)), k
