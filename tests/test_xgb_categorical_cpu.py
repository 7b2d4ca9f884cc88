"""CPU: xgboost default-left and categorical splits -- the plan compiler's node flags and category bitset section, its
refusals, the restated predictor's routing rule by rule, the srsnv k-fold step against the reference's own output, and
tests/test_gpu_xgb_categorical.py on the host emulation of the kernel sources."""
import os
import struct
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

from tests import xgb_categorical_ref as XR
from variantcalling_b200 import model_apply as MA
from variantcalling_b200 import model_compiler as MC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "host_emu")


def _doc(trees, n_features=2):
    return {"learner": {"objective": {"name": "binary:logistic"},
                        "learner_model_param": {"base_score": "0.5", "num_class": "0", "num_feature": str(n_features)},
                        "gradient_booster": {"name": "gbtree", "model": {"trees": trees, "tree_info": [0] * len(trees)}}}}


def _stump(feature=0, cond=0.5, default_left=0, cats=None, leaves=(-1.0, 1.0)):
    """Root split on `feature` with two leaves; `cats`: the root is categorical with that set."""
    tr = {"left_children": [1, -1, -1], "right_children": [2, -1, -1], "split_indices": [feature, 0, 0],
          "split_conditions": [cond, *leaves], "default_left": [default_left, 0, 0], "split_type": [0, 0, 0],
          "categories": [], "categories_nodes": [], "categories_segments": [], "categories_sizes": []}
    if cats is not None:
        tr.update(split_type=[1, 0, 0], split_conditions=[float("nan"), *leaves], categories=list(cats),
                  categories_nodes=[0], categories_segments=[0], categories_sizes=[len(cats)])
    return tr


def _sections(doc, n_features=2):
    """(nodes [(value bits, feature, right)], node flags, cat header (words, flagged), cat words) of a compiled forest."""
    m = MC._lower_xgboost_json(doc, n_features)  # noqa: SLF001
    sec, n_trees, n_nodes, n_rows = m["section"], m["n_trees"], m["n_nodes"], m["n_leaf_rows"]
    pad = lambda n: n + (-n % 8)  # noqa: E731
    off = pad(4 * (n_trees + 1)) + pad(n_trees)
    nodes = [struct.unpack_from("<IhH", sec, off + 8 * i) for i in range(n_nodes)]
    off += pad(8 * n_nodes) + pad(8 * n_rows)
    flags = list(sec[off:off + n_nodes])
    off += pad(n_nodes)
    n_words, n_flagged = struct.unpack_from("<II", sec, off)
    words = list(struct.unpack_from(f"<{n_words}I", sec, off + 8))
    return nodes, flags, (n_words, n_flagged), words


def test_compiler_writes_flags_and_bitsets():
    doc = _doc([_stump(cats=[1, 3, 40]), _stump(default_left=1), _stump()])
    nodes, flags, hdr, words = _sections(doc)
    # preorder per tree: root, left leaf, right leaf
    assert flags == [MC.NODE_CATEGORICAL, 0, 0, MC.NODE_DEFAULT_LEFT, 0, 0, 0, 0, 0]
    assert hdr == (2, 2) and words == [(1 << 1) | (1 << 3), 1 << 8]       # code 40: bit 8 of word 1
    assert nodes[0][0] == 0 | (2 << 24)                                      # UGVC_CAT_REF(first word 0, 2 words)
    assert struct.unpack("<f", struct.pack("<I", nodes[3][0]))[0] == 0.5    # a numeric node keeps its threshold
    sk = _sections(_doc([_stump(), _stump()]))
    assert sk[1] == [0] * 6 and sk[2] == (0, 0) and sk[3] == []


def test_compiler_refuses_malformed_category_sections():
    def bad(**upd):
        tr = _stump(cats=[2, 5])
        tr.update(upd)
        return _doc([tr])

    with pytest.raises(MC.PlanError, match="out of range"):
        MC.compile_plan_model_only(bad(categories_segments=[1]), 2)
    with pytest.raises(MC.PlanError, match="out of range"):
        MC.compile_plan_model_only(bad(categories_sizes=[0]), 2)
    with pytest.raises(MC.PlanError, match="missing from categories_nodes"):
        MC.compile_plan_model_only(bad(categories_nodes=[], categories_segments=[], categories_sizes=[]), 2)
    with pytest.raises(MC.PlanError, match="negative"):
        MC.compile_plan_model_only(bad(categories=[-1, 5]), 2)
    with pytest.raises(MC.PlanError, match="below 1024"):
        MC.compile_plan_model_only(bad(categories=[2, 1024]), 2)
    with pytest.raises(MC.PlanError, match="not a categorical split"):
        MC.compile_plan_model_only(bad(categories_nodes=[1]), 2)
    MC.compile_plan_model_only(bad(categories=[2, 1023]), 2)  # the largest code the limit allows


def test_restated_routing_rule_by_rule():
    """One row per rule on stumps: leaf -1 (left) or +1 (right)."""
    def side(tr, v):
        p1 = XR.predict_proba(_doc([tr]), np.array([[v, 0.0]], dtype=np.float32))[0, 1]
        return "L" if p1 < 0.5 else "R"

    nan = float("nan")
    assert side(_stump(default_left=1), nan) == "L" and side(_stump(default_left=0), nan) == "R"
    assert side(_stump(), 0.25) == "L" and side(_stump(), 0.5) == "R"                  # numeric: x < cond
    cat = _stump(cats=[0, 2, 7])
    assert side(cat, 2.0) == "R" and side(cat, 3.0) == "L"                              # in the set / not in it
    assert side(cat, 40.0) == "L"                                                        # past the bitset
    assert side(cat, -1.0) == "L" and side(cat, -0.5) == "L"                             # negative: invalid
    assert side(cat, 2.7) == "R" and side(cat, 7.99) == "R" and side(cat, 1.5) == "L"   # truncation
    assert side(cat, -0.0) == "R"                                                        # -0.0 is category 0
    assert side(_stump(cats=[0]), float(2 ** 24)) == "L"                                # >= 2^24: invalid
    assert side(_stump(cats=[0], default_left=1), nan) == "L" and side(_stump(cats=[0]), nan) == "R"


def test_frame_matrix_reads_frames_like_dmatrix():
    df = pd.DataFrame({"a": ["x", "y", None, "z"], "b": [1.5, np.nan, 3, 4],
                       "c": pd.array([1, None, 3, 4], dtype="Int64"), "d": [True, False, True, False]})
    df = MA.set_categorical_columns(df, {"a": ["y", "x"]})  # "z" is not a category: missing
    x = MA.frame_matrix(df, ["a", "b", "c", "d"])
    want = np.array([[1, 1.5, 1, 1], [0, np.nan, np.nan, 0], [np.nan, 3, 3, 1], [np.nan, 4, 4, 0]], dtype=np.float32)
    assert x.dtype == np.float32 and np.array_equal(x, want, equal_nan=True)
    with pytest.raises(ValueError, match="feature_names mismatch"):
        MA.frame_matrix(df, ["b", "a", "c", "d"])
    with pytest.raises(ValueError, match="dtype"):
        MA.frame_matrix(pd.DataFrame({"s": pd.Series(["u"], dtype=object)}))


def test_k_fold_matches_the_reference_golden():
    """tests/golden/srsnv_kfold.npz: the reference's k_fold_predict_proba on the two srsnv fold models (restated
    predictor behind them); the mirror with the same models gives the same values bit for bit."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "srsnv_kfold.npz"))
    features = XR.metadata_features()
    names = [f["name"] for f in features]
    df = MA.set_categorical_columns(XR.srsnv_frame(2024, g["x"].shape[0], features),
                                    {f["name"]: list(f["values"]) for f in features if f["type"] == "c"})
    assert np.array_equal(MA.frame_matrix(df[names], names), g["x"], equal_nan=True)
    df["fold_id"] = XR.srsnv_folds(7, df.shape[0])
    assert np.array_equal(df["fold_id"].to_numpy(), g["fold"], equal_nan=True)
    models = [XR.OracleModel(XR.load_golden_json(f"416119_L7402.test.model_fold_{k}.json")) for k in (0, 1)]
    got = MA.k_fold_predict_proba(models, df, names, 2)
    assert np.array_equal(got.to_numpy(), g["preds"], equal_nan=True)
    assert np.isnan(got[~df["fold_id"].isin([0, 1]) & df["fold_id"].notna()]).all()


def test_gpu_file_passes_on_the_host_emulation():
    build = subprocess.run(["make", "-C", EMU_DIR], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    env = dict(os.environ, UGVC_LIB_PATH=os.path.join(EMU_DIR, "_build", "libugvc_emu.so"))
    run = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                          "tests/test_gpu_xgb_categorical.py"], cwd=ROOT, env=env, capture_output=True, text=True,
                         timeout=3000)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0, tail
    assert " passed" in run.stdout and "failed" not in run.stdout.splitlines()[-1], tail
