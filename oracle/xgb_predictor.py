"""ORACLE (test infrastructure, not product code).

NumPy restatement of xgboost's CPU predictor for gbtree models (xgboost 2.1.2 is pinned by the
reference, ``ugbio_utils/src/core/pyproject.toml:38``, and called at
``ugbio_filtering/variant_filtering_utils.py:123-124``; the package is not installed here).

PARITY STATUS: unpinned against xgboost itself.  Published algorithm restated: for every row the
margin starts at logit(base_score) (binary:logistic) and the leaf values of the trees are added
in tree order in float32; a node sends a row left when ``x < split_condition`` (float32); the
probability is ``1 / (1 + exp(-margin))`` in float32 and ``predict_proba`` returns
``[1 - p, p]``.  Multi-class (multi:softprob) keeps one margin per class (tree_info gives the
class of each tree) and applies a float32 softmax.
"""
from __future__ import annotations

import numpy as np


def sklearn_gb_to_xgb_json(model) -> dict:
    """Re-express a fitted sklearn GradientBoostingClassifier as an xgboost JSON model document
    (same trees, xgboost's conventions) -- a way to get a realistic xgboost-format model without
    xgboost: ``x <= t`` (sklearn, t float64) becomes ``x < t'`` with t' the float32 just above
    floor32(t); leaf values are learning_rate * value rounded to float32."""
    k = len(model.classes_)
    n_out = model.estimators_.shape[1]
    trees, info = [], []
    for stage in range(model.estimators_.shape[0]):
        for o in range(n_out):
            t = model.estimators_[stage, o].tree_
            thr = t.threshold.astype(np.float64)
            f = thr.astype(np.float32)
            too_big = f.astype(np.float64) > thr
            f[too_big] = np.nextafter(f[too_big], np.float32(-np.inf))
            cond = np.nextafter(f, np.float32(np.inf))
            leaf = (np.float64(model.learning_rate) * t.value[:, 0, 0]).astype(np.float32)
            is_leaf = t.children_left == -1
            cond = np.where(is_leaf, leaf, cond).astype(np.float32)
            trees.append({"left_children": t.children_left.tolist(), "right_children": t.children_right.tolist(),
                          "split_indices": np.where(is_leaf, 0, t.feature).tolist(),
                          "split_conditions": [float(v) for v in cond], "default_left": [0] * t.node_count,
                          "base_weights": [float(v) for v in cond]})
            info.append(o)
    objective = "binary:logistic" if k == 2 else "multi:softprob"
    base_score = 0.5
    if k == 2:  # carry sklearn's prior: margin0 = logit(base_score) = the boosting init
        init = float(np.asarray(model._raw_predict_init(np.zeros((1, model.n_features_in_)))).ravel()[0])  # noqa: SLF001
        base_score = 1.0 / (1.0 + np.exp(-init))
    return {"learner": {"objective": {"name": objective},
                        "learner_model_param": {"base_score": repr(float(base_score)), "num_class": str(0 if k == 2 else k),
                                                "num_feature": str(model.n_features_in_)},
                        "gradient_booster": {"name": "gbtree", "model": {"trees": trees, "tree_info": info}}}}


def random_gbtree_document(seed: int, x: np.ndarray, n_trees: int, *, num_class: int = 0, max_depth: int = 12,
                           full_depth: bool = False, leaf_p: float = 0.3, tree_info="rounds",
                           base_score: float = 0.5) -> dict:
    """A random xgboost gbtree JSON document over the columns of ``x`` -- deep / large models without xgboost.

    ``num_class`` 0 gives ``binary:logistic``, otherwise ``multi:softprob`` with that many classes (2 included).
    Every tree has its own depth in [1, max_depth] (exactly ``max_depth`` with ``full_depth``), reached by one
    random root-to-leaf path; off that path a node becomes a leaf with probability ``leaf_p``, so the trees are
    unbalanced.  Nodes are numbered breadth first like xgboost's.  A split condition is a float32 value of its
    column in ``x`` (rows then sit exactly on it); leaf values are float32.  ``tree_info``: "rounds" (class of
    tree t = t % num_class, xgboost's layout), "blocks" (all trees of class 0, then class 1, ...), "shuffled" (a
    seeded permutation of the rounds layout) or an explicit list."""
    rng = np.random.default_rng(seed)
    x = np.asarray(x, dtype=np.float32)
    n_out = max(1, num_class)
    trees = []
    for _ in range(n_trees):
        depth = max_depth if full_depth else int(rng.integers(1, max_depth + 1))
        path = rng.integers(0, 2, size=depth)  # the branch taken at each level by the path that reaches `depth`
        left, right, feat, cond = [], [], [], []
        queue = [(0, True)]  # (level, on the deep path); index in the lists == breadth-first node id
        left.append(-1), right.append(-1), feat.append(0), cond.append(0.0)
        head = 0
        while head < len(queue):
            level, on_path = queue[head]
            nid = head
            head += 1
            is_leaf = level == depth or (not on_path and rng.random() < leaf_p)
            if is_leaf:
                cond[nid] = float(np.float32(rng.normal(0.0, 0.4)))
                continue
            f = int(rng.integers(0, x.shape[1]))
            feat[nid] = f
            cond[nid] = float(x[int(rng.integers(0, x.shape[0])), f])
            for side in (0, 1):
                child = len(left)
                left.append(-1), right.append(-1), feat.append(0), cond.append(0.0)
                queue.append((level + 1, on_path and int(path[level]) == side))
                if side == 0:
                    left[nid] = child
                else:
                    right[nid] = child
        trees.append({"left_children": left, "right_children": right, "split_indices": feat,
                      "split_conditions": cond, "default_left": [0] * len(left), "base_weights": list(cond)})
    if isinstance(tree_info, str):
        rounds = [t % n_out for t in range(n_trees)] if num_class else [0] * n_trees
        if tree_info == "rounds":
            tree_info = rounds
        elif tree_info == "blocks":
            tree_info = sorted(rounds)
        elif tree_info == "shuffled":
            tree_info = [int(v) for v in rng.permutation(rounds)]
        else:
            raise ValueError(tree_info)
    objective = "multi:softprob" if num_class else "binary:logistic"
    return {"learner": {"objective": {"name": objective},
                        "learner_model_param": {"base_score": repr(float(base_score)), "num_class": str(num_class),
                                                "num_feature": str(x.shape[1])},
                        "gradient_booster": {"name": "gbtree", "model": {"trees": trees, "tree_info": list(tree_info)}}}}


def _expf(v: np.ndarray) -> np.ndarray:
    """libm's expf as xgboost's Sigmoid / Softmax call it: glibc's is correctly rounded for all but about one
    argument in 10^7, NumPy's SIMD float32 exp is not -- so: float64 exp, rounded once."""
    return np.exp(np.asarray(v, dtype=np.float32).astype(np.float64)).astype(np.float32)


def predict_proba(doc: dict, x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.float32)
    learner = doc["learner"]
    objective = learner["objective"]["name"]
    base_score = np.float32(float(learner["learner_model_param"]["base_score"]))
    model = learner["gradient_booster"]["model"]
    n_class = int(learner["learner_model_param"].get("num_class", "0"))
    n_out = 1 if objective == "binary:logistic" else n_class
    n = x.shape[0]
    if objective == "binary:logistic":
        init = np.float32(-np.log(np.float32(1.0) / base_score - np.float32(1.0)))
    else:
        init = base_score
    margin = np.full((n, n_out), init, dtype=np.float32)
    rows = np.arange(n)
    for ti, tr in enumerate(model["trees"]):
        left = np.asarray(tr["left_children"])
        right = np.asarray(tr["right_children"])
        feat = np.asarray(tr["split_indices"])
        cond = np.asarray(tr["split_conditions"], dtype=np.float32)
        node = np.zeros(n, dtype=np.int64)
        active = left[node] != -1
        while active.any():
            go_left = x[rows, feat[node]] < cond[node]
            nxt = np.where(go_left, left[node], right[node])
            node = np.where(active, nxt, node)
            active = left[node] != -1
        o = model["tree_info"][ti] if n_out > 1 else 0
        margin[:, o] = (margin[:, o] + cond[node]).astype(np.float32)
    if n_out == 1:
        p1 = (np.float32(1.0) / (np.float32(1.0) + _expf(-margin[:, 0]))).astype(np.float32)
        return np.stack([np.float32(1.0) - p1, p1], axis=1)
    mx = margin.max(axis=1, keepdims=True)
    e = _expf(margin - mx)
    s = e.astype(np.float64).sum(axis=1, keepdims=True)
    return (e / s.astype(np.float32)).astype(np.float32)
