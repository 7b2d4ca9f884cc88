"""ORACLE (test infrastructure, not product code): xgboost's CPU predictor with missing-value and categorical routing.

NumPy restatement of xgboost 2.1.2's ``GetNextNode`` / ``common::Decision`` (the version the reference pins, not
installed here: PARITY UNPINNED), on top of the plain restatement in ``oracle/xgb_predictor.py`` (same margins in
float32 in tree order, same float32 sigmoid / softmax):

* NaN goes to the node's default child (``default_left[n]``: left, else right), at every node;
* a numeric node sends ``x < split_conditions[n]`` (float32) left;
* a categorical node (``split_type[n] == 1``; its set ``categories[categories_segments[i]:][:categories_sizes[i]]``
  for ``categories_nodes[i] == n``) sends an invalid category (``x < 0`` or ``x >= 2^24``) left, ``int(x)``
  (truncated) past the node's bitset left, a category in the set right and one not in it left.

Also a generator of categorical / default-left documents without xgboost (``categorical_document``) and an
oracle-driven stand-in for a fitted classifier (``OracleModel``) for the k-fold step.
"""
from __future__ import annotations

import ast
import gzip
import json
import os

import numpy as np
import pandas as pd

from oracle import xgb_predictor as XP
from variantcalling_b200 import model_apply as MA

MAX_CAT = 1 << 24  # xgboost's InvalidCat bound
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def node_sets(tr) -> dict:
    """node id -> (category codes, bitset words) of one tree's categorical nodes (xgboost sizes the bitset from the
    largest code: ceil((max + 1) / 32) words)."""
    out = {}
    cats = tr.get("categories", [])
    for nid, seg, size in zip(tr.get("categories_nodes", []), tr.get("categories_segments", []), tr.get("categories_sizes", [])):
        codes = np.asarray(cats[seg:seg + size], dtype=np.int64)
        out[int(nid)] = (codes, (int(codes.max()) + 1 + 31) // 32)
    return out


def go_left(tr, node: np.ndarray, v: np.ndarray, sets: dict) -> np.ndarray:
    """The routing decision of the rows sitting on ``node`` with feature values ``v`` (float32)."""
    n_nodes = len(tr["left_children"])
    dl = np.asarray(tr.get("default_left") or [0] * n_nodes, dtype=np.int64)[node] != 0
    cat = np.asarray(tr.get("split_type") or [0] * n_nodes, dtype=np.int64)[node] == 1
    cond = np.asarray(tr["split_conditions"], dtype=np.float32)[node]
    with np.errstate(invalid="ignore"):
        numeric_left = v < cond
        invalid = (v < 0) | (v >= np.float32(MAX_CAT))
    cat_left = np.ones(v.shape, dtype=bool)
    for nid in np.unique(node[cat]):
        m = cat & (node == nid) & ~np.isnan(v) & ~invalid
        codes, words = sets[int(nid)]
        c = np.trunc(v[m]).astype(np.int64)
        inside = c < words * 32
        cat_left[m] = ~(inside & np.isin(c, codes))
    return np.where(np.isnan(v), dl, np.where(cat, cat_left, numeric_left))


def predict_proba(doc: dict, x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.float32)
    learner = doc["learner"]
    objective = learner["objective"]["name"]
    base_score = np.float32(float(learner["learner_model_param"]["base_score"]))
    model = learner["gradient_booster"]["model"]
    n_class = int(learner["learner_model_param"].get("num_class", "0"))
    n_out = 1 if objective == "binary:logistic" else n_class
    n = x.shape[0]
    init = np.float32(-np.log(np.float32(1.0) / base_score - np.float32(1.0))) if n_out == 1 else base_score
    margin = np.full((n, n_out), init, dtype=np.float32)
    rows = np.arange(n)
    for ti, tr in enumerate(model["trees"]):
        left = np.asarray(tr["left_children"])
        right = np.asarray(tr["right_children"])
        feat = np.asarray(tr["split_indices"])
        cond = np.asarray(tr["split_conditions"], dtype=np.float32)
        sets = node_sets(tr)
        node = np.zeros(n, dtype=np.int64)
        active = left[node] != -1
        while active.any():
            a = np.flatnonzero(active)
            gl = go_left(tr, node[a], x[rows[a], feat[node[a]]], sets)
            node[a] = np.where(gl, left[node[a]], right[node[a]])
            active = left[node] != -1
        o = model["tree_info"][ti] if n_out > 1 else 0
        margin[:, o] = (margin[:, o] + cond[node]).astype(np.float32)
    if n_out == 1:
        p1 = (np.float32(1.0) / (np.float32(1.0) + XP._expf(-margin[:, 0]))).astype(np.float32)  # noqa: SLF001
        return np.stack([np.float32(1.0) - p1, p1], axis=1)
    mx = margin.max(axis=1, keepdims=True)
    e = XP._expf(margin - mx)  # noqa: SLF001
    s = e.astype(np.float64).sum(axis=1, keepdims=True)
    return (e / s.astype(np.float32)).astype(np.float32)


def categorical_document(seed: int, x: np.ndarray, n_trees: int, cat_features, *, n_codes: int = 14, cat_p: float = 0.7,
                         default_left_p: float = 0.5, wide_p: float = 0.1, **kw) -> dict:
    """``oracle.xgb_predictor.random_gbtree_document`` (same options in ``kw``) with random ``default_left`` on every
    internal node and, with probability ``cat_p``, a categorical split at an internal node on a column of
    ``cat_features``: a set of 1 to n_codes - 1 codes below ``n_codes``, or (probability ``wide_p``) one that also
    holds a code in [256, 1024), so the node's bitset is long and most codes fall inside it unset."""
    doc = XP.random_gbtree_document(seed, x, n_trees, **kw)
    rng = np.random.default_rng(seed + 7919)
    cat_features = set(int(f) for f in cat_features)
    for tr in doc["learner"]["gradient_booster"]["model"]["trees"]:
        n_nodes = len(tr["left_children"])
        st, dl = [0] * n_nodes, [0] * n_nodes
        cats, c_nodes, c_seg, c_size = [], [], [], []
        for nid in range(n_nodes):
            if tr["left_children"][nid] == -1:
                continue
            dl[nid] = int(rng.random() < default_left_p)
            if tr["split_indices"][nid] in cat_features and rng.random() < cat_p:
                size = int(rng.integers(1, n_codes))
                codes = sorted(int(c) for c in rng.choice(n_codes, size=size, replace=False))
                if rng.random() < wide_p:
                    codes.append(int(rng.integers(256, 1024)))
                st[nid] = 1
                tr["split_conditions"][nid] = float("nan")
                c_nodes.append(nid), c_seg.append(len(cats)), c_size.append(len(codes))
                cats.extend(codes)
        tr.update(split_type=st, default_left=dl, categories=cats, categories_nodes=c_nodes,
                  categories_segments=c_seg, categories_sizes=c_size)
    return doc


class OracleModel:
    """A fitted classifier stand-in: ``predict_proba(frame)`` reads the frame as xgboost's DMatrix does
    (``model_apply.frame_matrix``) and returns the restatement's float32 probabilities, as xgboost returns them."""

    def __init__(self, doc: dict):
        self.doc = doc
        self.feature_names = doc["learner"].get("feature_names") or None

    def predict_proba(self, x):
        if hasattr(x, "columns"):
            x = MA.frame_matrix(x, self.feature_names)
        return predict_proba(self.doc, x)


# ---- the srsnv fixtures (tests/golden: the reference's fold models and their metadata; scripts/make_golden_srsnv.py)
def load_golden_json(name: str) -> dict:
    with gzip.open(os.path.join(GOLDEN, name + ".gz")) as fh:
        return json.load(fh)


def metadata_features() -> list:
    """[{name, type ('c' / 'int' / 'float'), values (category -> code)}] of the srsnv fold models, in model order."""
    meta = load_golden_json("416119_L7402.test.srsnv_metadata.json")
    return ast.literal_eval(meta["features"]) if isinstance(meta["features"], str) else meta["features"]


def srsnv_frame(seed: int, n: int, features) -> pd.DataFrame:
    """Raw values of the model's features: strings for categorical columns (some outside the fitted categories),
    numbers with NaNs."""
    rng = np.random.default_rng(seed)
    cols = {}
    for f in features:
        if f["type"] == "c":
            vals = list(f["values"]) + ["UNSEEN", "N"]
            cols[f["name"]] = pd.Series(rng.choice(np.array(vals, dtype=object), n), dtype=object)
        else:
            v = np.round(rng.gamma(2.0, 20.0, n)) if f["type"] == "int" else rng.random(n)
            v[rng.random(n) < 0.05] = np.nan
            cols[f["name"]] = v
    return pd.DataFrame(cols)


def srsnv_folds(seed: int, n: int) -> np.ndarray:
    """Fold ids of two-fold inference: valid (0, 1), none (NaN) and out of range (-1, 2, 5)."""
    rng = np.random.default_rng(seed)
    return rng.choice(np.array([0, 1, np.nan, -1, 2, 5]), n, p=[0.35, 0.35, 0.2, 0.04, 0.03, 0.03])
