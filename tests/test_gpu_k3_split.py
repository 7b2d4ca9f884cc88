"""GPU: k3_heap_split (two threads per record, the second one's leaf rows handed over and added after the first one's)
against the one-thread k3_heap on the same rows, bit for bit: the split keeps every sum's order, so FILTER, the fp32
and fp64 probabilities and qual are identical.  Each side runs in a child process (UGVC_K3_SHAPE is read once per
process): shape 9 is the split form, shape 7 the one-thread k3_heap with the smallest tile.  Models cover odd tree
counts and counts not divisible by the eight chains, fewer trees than chains, depths 1-8, random forests, multi-class
boosting, xgboost default-left and categorical nodes; record counts leave partial tiles and partial waves."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import xgb_predictor as XP
from tests import util
from tests import xgb_categorical_ref as XR
from variantcalling_b200 import model_compiler as MC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPLIT, ONE = "9", "7"

_CHILD = r"""
import json, sys
import numpy as np
from variantcalling_b200 import lib
mode, blob, inp, out, ns = sys.argv[1], open(sys.argv[2], "rb").read(), sys.argv[3], sys.argv[4], json.loads(sys.argv[5])
c = lib.Context(0)
c.enable_phreds(2)
c.load_plan(blob)
res = {}
if mode == "x":
    x = np.load(inp)
    c.reserve(4096, x.shape[0], 1)
    cfg = c.k3_config()
    for n in ns or [x.shape[0]]:
        c.counts_reset()
        r = c.predict_features(x[:n], threshold=20.0)
        cnt = c.counts()
        res[f"{n}"] = np.concatenate([r["low_score"].view(np.uint8), r["probs"].view(np.uint8).ravel(), r["qual"].view(np.uint8),
                                      c.collect_phreds(0, n).view(np.uint8).ravel(),
                                      np.array([cnt["n_records"], cnt["n_low_score"], cnt["n_pass"]], np.int64).view(np.uint8)])
else:
    text = open(inp, "rb").read()
    c.set_key_order(*lib.learn_key_order(text))
    c.reserve(len(text) + 4096, text.count(b"\n") + 16, 1)
    cfg = c.k3_config()
    r = c.filter_batch(text, 30.0)
    n = r["n_records"]
    res["vcf"] = np.concatenate([r["low_score"].view(np.uint8), r["probs"].view(np.uint8).ravel(), r["qual"].view(np.uint8),
                                 c.collect_phreds(0, n).view(np.uint8).ravel(), c.debug_features(n).view(np.uint8).ravel()])
np.savez(out, **res)
print(json.dumps(cfg))
c.close()
"""


def _child(tmp_path, shape, mode, blob, inp, ns=()):
    tag = f"{shape}_{len(os.listdir(tmp_path))}"
    bp, op = tmp_path / f"plan_{tag}.bin", tmp_path / f"out_{tag}.npz"
    bp.write_bytes(blob)
    env = dict(os.environ, UGVC_K3_SHAPE=shape)
    r = subprocess.run([sys.executable, "-c", _CHILD, mode, str(bp), str(inp), str(op), json.dumps(list(ns))], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1]), dict(np.load(op))


def _rows(seed, f, n=1500, nan=True):
    """Rows with ties on integer thresholds; 3 % NaN (missing values) for xgboost models, which take them."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, f)).astype(np.float32)
    x[:, ::5] = np.round(x[:, ::5] * 3)
    if nan:
        x[rng.random(x.shape) < 0.03] = np.nan
    return x


def _train(seed, f, k, n=800):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, f))
    s = x[:, 0] - 0.7 * x[:, 1] + 0.5 * x[:, 2] * x[:, 3] + rng.normal(0, 1.0, n)
    return x, np.digitize(s, np.quantile(s, np.linspace(0, 1, k + 1)[1:-1]))


def _gb(k, n_estimators, depth, f=20):
    from sklearn.ensemble import GradientBoostingClassifier

    x, y = _train(depth, f, k)
    return GradientBoostingClassifier(n_estimators=n_estimators, max_depth=depth, learning_rate=0.2, subsample=0.5,
                                      random_state=0).fit(x, y)


def _rf(k, n_estimators, depth, f=20):
    from sklearn.ensemble import RandomForestClassifier

    x, y = _train(depth + 100, f, k)
    return RandomForestClassifier(n_estimators=n_estimators, max_depth=depth, random_state=0, n_jobs=1).fit(x, y)


def _xgb(n_trees, depth, num_class=0, f=20):
    return XP.random_gbtree_document(n_trees, _rows(n_trees, f, 400), n_trees, num_class=num_class, max_depth=depth)


def _xgb_cat(n_trees, depth, f=24):
    rng = np.random.default_rng(n_trees)
    base = rng.normal(0, 1, size=(400, f)).astype(np.float32)
    cats = list(range(0, f, 3))
    base[:, cats] = rng.integers(0, 14, size=(400, len(cats)))
    return XR.categorical_document(n_trees, base, n_trees, cats, max_depth=depth, leaf_p=0.2), cats


# name -> (model builder, n_features)
CASES = {
    "gb2_67x1": (lambda: _gb(2, 67, 1), 20),
    "gb2_67x3": (lambda: _gb(2, 67, 3), 20),
    "gb2_101x6": (lambda: _gb(2, 101, 6), 20),
    "gb2_67x8": (lambda: _gb(2, 67, 8), 20),
    "gb2_5x4_fewer_than_chains": (lambda: _gb(2, 5, 4), 20),
    "gb2_1x2_one_tree": (lambda: _gb(2, 1, 2), 20),
    "gb3_23x5_multiclass": (lambda: _gb(3, 23, 5), 20),
    "rf3_33x6": (lambda: _rf(3, 33, 6), 20),
    "rf2_70x7": (lambda: _rf(2, 70, 7), 20),
    "xgb2_77x6_default_left": (lambda: _xgb(77, 6), 20),
    "xgbm3_45x5": (lambda: _xgb(45, 5, num_class=3), 20),
}


@pytest.mark.parametrize("name", list(CASES))
def test_split_equals_one_thread_per_record(tmp_path, name):
    build, f = CASES[name]
    model = build()
    blob = MC.compile_plan_model_only(model, f).blob
    x = _rows(len(name), f, nan=isinstance(model, dict))
    xp = tmp_path / "x.npy"
    np.save(xp, x)
    cfg_s, _ = _child(tmp_path, SPLIT, "x", blob, xp, [1])
    assert (cfg_s["kernel"], cfg_s["split"], cfg_s["resident"]) == ("heap", 2, True), cfg_s
    gs, wave = cfg_s["gs"], cfg_s["grid"] * cfg_s["groups"] * cfg_s["gs"]
    n_full = max(x.shape[0], wave + 1)
    xf = np.resize(x, (n_full, f))
    np.save(xp, xf)
    ns = sorted({1, gs - 1, gs, gs + 1, 2 * gs + 7, wave - 1, wave, n_full})
    cfg_s, split = _child(tmp_path, SPLIT, "x", blob, xp, ns)
    cfg_o, one = _child(tmp_path, ONE, "x", blob, xp, ns)
    assert cfg_o["split"] == 1 and cfg_o["tpb"] == 128, cfg_o
    for n in ns:
        assert np.array_equal(split[str(n)], one[str(n)]), n


def test_split_equals_one_thread_per_record_categorical(tmp_path):
    doc, cats = _xgb_cat(71, 6)
    f = 24
    blob = MC.compile_plan_model_only(doc, f).blob
    rng = np.random.default_rng(3)
    x = _rows(4, f, 3000)
    x[:, cats] = rng.choice(np.array([*range(14), np.nan, -1.0, 2.5, 40.0], np.float32), size=(3000, len(cats)))
    xp = tmp_path / "x.npy"
    np.save(xp, x)
    cfg_s, split = _child(tmp_path, SPLIT, "x", blob, xp, [1, 159, 160, 161, 3000])
    cfg_o, one = _child(tmp_path, ONE, "x", blob, xp, [1, 159, 160, 161, 3000])
    assert (cfg_s["split"], cfg_s["walk"]) == (2, "categorical") and cfg_o["split"] == 1, (cfg_s, cfg_o)
    for k in split:
        assert np.array_equal(split[k], one[k]), k


def test_split_assembles_the_features_from_vcf_records(tmp_path):
    """The VCF entry point: the pair assembles the record's features from K1's slots (the transformer's policies) in
    two halves, then scores; the default choice for a tile-limited plan of 64 trees or more is the split form."""
    from sklearn.ensemble import GradientBoostingClassifier

    from variantcalling_b200.vcf_header import VcfHeader

    ds = util.make_dataset(n_records=3000, n_custom=40, seed=23)
    _, tr, x = util.fit_transformer(ds)
    model = GradientBoostingClassifier(n_estimators=100, max_depth=6, learning_rate=0.15, subsample=0.4,
                                       random_state=0).fit(x, ds["labels"])
    blob = MC.compile_plan(VcfHeader(ds["header_text"]), tr, model, ds["customs"]).blob
    vp = tmp_path / "in.vcf"
    vp.write_bytes(ds["text"] if isinstance(ds["text"], bytes) else ds["text"].encode())
    cfg_d, auto = _child(tmp_path, "-1", "vcf", blob, vp)
    cfg_s, split = _child(tmp_path, SPLIT, "vcf", blob, vp)
    cfg_o, one = _child(tmp_path, ONE, "vcf", blob, vp)
    assert cfg_s["split"] == 2 and cfg_o["split"] == 1
    # 81 features, 100 trees of depth 6 (the bench's plan shape): 512/2 does not hold it, so the split form is the default
    assert x.shape[1] == 81 and cfg_d == cfg_s, (cfg_d, cfg_s)
    assert np.array_equal(split["vcf"], one["vcf"]) and np.array_equal(auto["vcf"], one["vcf"])
