"""Plan compiler: (VCF header, fitted transformer, model) -> flat plan blob.

The reference keeps the feature spec as a fitted sklearn ``ColumnTransformer`` and
the classifier as an ``XGBClassifier`` inside one pickle
(``ugbio_utils/src/filtering/ugbio_filtering/train_models_pipeline.py:151-160``,
read at ``filter_variants_pipeline.py:89-94``).  The CUDA kernels cannot run
Python callables, so this module lowers the *fitted* objects:

* every ColumnTransformer entry (``transformers.py:221-344``) becomes raw-slot
  requests for K1 (which tag, which element, which string reducer) and per-column
  missing/absent policies for K2, reproducing what the reference's Python
  function does to ``None`` / ``(None,)`` / short tuples / unknown strings;
* fitted ``OrdinalEncoder`` categories become K1 dictionaries;
* the classifier becomes a flat model section: sklearn ``LogisticRegression``
  (fp64), ``GradientBoostingClassifier`` / ``RandomForestClassifier`` (preorder
  node arrays, fp64 leaves, thresholds rounded *down* to fp32 so ``x <= t``
  decides identically on fp32 inputs) or an xgboost JSON model dump
  (``x < t``, fp32 margins).

Entries are recognised by type and by ``func.__name__`` so a pickle produced by the
reference's own ``ugbio_filtering.transformers`` lowers the same way as one
produced by ``variantcalling_b200.transformers``.  Anything this compiler cannot
lower exactly raises ``PlanError`` -- there is no approximate or CPU fallback.

Binary layout: ``variantcalling_b200/csrc/plan.h``.
"""
from __future__ import annotations

import json
import struct
from dataclasses import dataclass, field

import numpy as np

from variantcalling_b200.vcf_header import VcfHeader

PLAN_MAGIC = 0x50564755
PLAN_VERSION = 9
MAX_TAGS, MAX_SLOTS, MAX_FEATURES, MAX_CLASSES, NAME_MAX = 128, 250, 250, 4, 32
MAX_DICTS, MAX_STRINGS = 64, 96

KIND_INT, KIND_FLOAT, KIND_STR, KIND_FLAG, KIND_SCALAR = 1, 2, 3, 4, 8
(RED_NUM, RED_BASE, RED_INSDEL, RED_DICT, RED_MOTIF_L, RED_MOTIF_R, RED_STRNUM, RED_GT_HOM, RED_LEN,
 RED_REGION) = range(10)
RED_FIX_QUAL, RED_FIX_ALLELE0, RED_FIX_ALLELE1, RED_FIX_INDEL, RED_FIX_NALLELES = 16, 17, 18, 19, 20
TAG_FIXED, ELEM_WHOLE = 0xFF, 0xFF
POL_VALUE, POL_ERROR, POL_NULL = 0, 1, 2
MODEL_LOGISTIC, MODEL_GB_SKLEARN, MODEL_RF_SKLEARN, MODEL_XGB = 1, 2, 3, 4
CMP_LE, CMP_LT = 0, 1
NODE_DEFAULT_LEFT, NODE_CATEGORICAL = 1, 2
MAX_CATEGORIES = 1024  # category codes in [0, 1024): a node's bitset has at most 32 words (plan.h UGVC_MAX_CATEGORIES)


class PlanError(ValueError):
    """The model / transformer / header combination cannot be lowered exactly."""


# --------------------------------------------------------------------------- helpers
def _kind(number: str, vtype: str) -> int:
    base = {"Integer": KIND_INT, "Float": KIND_FLOAT, "String": KIND_STR, "Character": KIND_STR,
            "Flag": KIND_FLAG}.get(vtype)
    if base is None:
        raise PlanError(f"unknown VCF Type {vtype!r}")
    return base | (KIND_SCALAR if number == "1" else 0)


def _pad8(b: bytes) -> bytes:
    return b + b"\0" * (-len(b) % 8)


@dataclass
class _SlotReq:
    tag: str | None          # VCF tag, or None for a fixed column
    elem: int
    reducer: int
    dict_id: int = 0


@dataclass
class _Feature:
    slot: _SlotReq
    absent: tuple            # (policy, value)
    missing: tuple


@dataclass
class Plan:
    blob: bytes
    n_features: int
    n_classes: int
    n_slots: int
    tags: list
    feature_names: list
    model_kind: int
    classes: list = field(default_factory=list)


def _describe(trans) -> list[str]:
    """Flatten one ColumnTransformer entry into a list of step descriptors."""
    from sklearn.impute import SimpleImputer
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import FunctionTransformer, OrdinalEncoder

    if isinstance(trans, str):
        return [trans]
    if isinstance(trans, Pipeline):
        out = []
        for _, step in trans.steps:
            out.extend(_describe(step))
        return out
    if isinstance(trans, FunctionTransformer):
        if trans.func is None:  # a fitted ColumnTransformer stores "passthrough" as an identity transformer
            return ["passthrough"]
        return ["fn:" + getattr(trans.func, "__name__", "?")]
    if isinstance(trans, SimpleImputer):
        if trans.strategy != "constant":
            raise PlanError(f"SimpleImputer strategy {trans.strategy!r} is not lowered")
        mv = trans.missing_values
        mv_name = "none" if mv is None else ("nan" if isinstance(mv, float) and np.isnan(mv) else repr(mv))
        return [f"impute:{mv_name}:{trans.fill_value!r}"]
    if isinstance(trans, OrdinalEncoder):
        return ["ordinal"]
    raise PlanError(f"transformer step {type(trans).__name__} is not lowered")


class _Builder:
    def __init__(self, header: VcfHeader, custom_info_fields):
        self.header = header
        self.col2tag = header.loader_columns(custom_info_fields)
        self.features: list[_Feature] = []
        self.feature_names: list[str] = []
        self.checks: list[tuple[_SlotReq, int, float]] = []
        self.combines: list[tuple[int, _SlotReq]] = []  # (feature index, second slot): max, nulls skipped
        self.dicts: list[list[str]] = []

    # ---- tag typing
    def kinds(self, tag: str) -> tuple[int, int]:
        ik = _kind(*self.header.info[tag]) if tag in self.header.info else 0
        fk = _kind(*self.header.formats[tag]) if tag in self.header.formats else 0
        if tag == "GT" and fk:
            fk = KIND_STR | KIND_SCALAR  # htslib decodes GT specially; K1 sees its text
        return ik, fk

    def tag_of(self, col: str) -> str:
        if col not in self.col2tag:
            raise PlanError(
                f"column {col!r} is needed by the transformer but no such INFO/FORMAT tag is declared in the "
                f"VCF header (the reference loader would drop it and the transformer would raise)")
        return self.col2tag[col]

    def _all_kinds(self, tag):
        return [k for k in self.kinds(tag) if k]

    def require(self, tag, *, scalar: bool | None, types: tuple):
        for k in self._all_kinds(tag):
            if (k & 7) == KIND_FLAG:
                raise PlanError(f"tag {tag}: Flag typed tags are not lowered as features")
            if (k & 7) not in types:
                raise PlanError(f"tag {tag}: header Type does not fit the transformer applied to it")
            if scalar is not None and bool(k & KIND_SCALAR) != scalar:
                want = "Number=1" if scalar else "a vector Number"
                raise PlanError(f"tag {tag}: the transformer applied to it needs {want} in the header")

    def add(self, name, slot, absent, missing):
        self.features.append(_Feature(slot, absent, missing))
        self.feature_names.append(name)

    def add_dict(self, cats) -> int:
        strs = []
        for c in cats:
            if not isinstance(c, str):
                raise PlanError(f"OrdinalEncoder category {c!r} is not a string")
            if len(c.encode()) > 24:  # noqa: PLR2004
                raise PlanError(f"category string {c!r} longer than 24 bytes")
            strs.append(c)
        if strs in self.dicts:
            return self.dicts.index(strs)
        self.dicts.append(strs)
        return len(self.dicts) - 1

    # ---- one ColumnTransformer entry -> features
    def lower_entry(self, name: str, trans, cols, width: int):  # noqa: C901, PLR0912, PLR0915
        steps = _describe(trans)
        col_list = [cols] if isinstance(cols, str) else list(cols)
        V, E = POL_VALUE, POL_ERROR
        NUM = (KIND_INT, KIND_FLOAT)

        def single_col():
            if len(col_list) != 1:
                raise PlanError(f"entry {name!r}: expected one input column")
            return col_list[0]

        if steps == ["drop"]:
            return
        if steps == ["passthrough"]:
            for col in col_list:
                if col == "indel":
                    self.add(col, _SlotReq(None, 0, RED_FIX_INDEL), (V, 0.0), (V, 0.0))
                elif col == "qual":
                    self.add(col, _SlotReq(None, 0, RED_FIX_QUAL), (E, 0.0), (E, 0.0))
                else:
                    tag = self.tag_of(col)
                    self.require(tag, scalar=True, types=NUM)
                    self.add(col, _SlotReq(tag, 0, RED_NUM), (E, 0.0), (E, 0.0))
            return
        if len(steps) == 1 and steps[0].startswith("impute:nan:"):
            fill = float(eval(steps[0].split(":", 2)[2]))  # noqa: S307  (repr of a number)
            for col in col_list:
                if col == "qual":
                    self.add(col, _SlotReq(None, 0, RED_FIX_QUAL), (V, fill), (V, fill))
                    continue
                tag = self.tag_of(col)
                self.require(tag, scalar=True, types=NUM)
                self.add(col, _SlotReq(tag, 0, RED_NUM), (V, fill), (V, fill))
            return
        head = steps[0]
        if head == "fn:tuple_encode_df":
            tag = self.tag_of(single_col())
            rest = steps[1:]
            kinds = self._all_kinds(tag)
            vector = [not (k & KIND_SCALAR) for k in kinds]
            if rest in ([], ["impute:nan:0"]):
                self.require(tag, scalar=None, types=NUM)
                # tuple -> first element (None -> NaN: a null unless imputed); scalar None -> 0
                miss_tuple = (V, 0.0) if rest else (E, 0.0)
                if any(vector) and not all(vector):
                    raise PlanError(f"tag {tag}: INFO and FORMAT declare different Number shapes")
                missing = miss_tuple if all(vector) else (V, 0.0)
                self.add(name, _SlotReq(tag, 0, RED_NUM), (V, 0.0), missing)
                return
            self.require(tag, scalar=False, types=(KIND_STR,))
            if rest == ["fn:allele_encode_single"]:
                self.add(name, _SlotReq(tag, 0, RED_BASE), (V, 0.0), (V, 0.0))
                return
            if rest == ["fn:ins_del_encode_df"]:
                self.add(name, _SlotReq(tag, 0, RED_INSDEL), (E, 0.0), (E, 0.0))
                return
            if rest == ["ordinal"]:
                enc = trans.steps[-1][1]
                if not hasattr(enc, "categories_"):
                    raise PlanError(f"entry {name!r}: the OrdinalEncoder is not fitted")
                did = self.add_dict(list(enc.categories_[0]))
                self.add(name, _SlotReq(tag, 0, RED_DICT, did), (E, 0.0), (E, 0.0))
                return
            raise PlanError(f"entry {name!r}: pipeline {steps} is not lowered")
        if steps == ["fn:tuple_encode_doublet_df"]:
            tag = self.tag_of(single_col())
            self.require(tag, scalar=False, types=NUM)
            for e in range(2):
                self.add(f"{name}_{e}", _SlotReq(tag, e, RED_NUM), (E, 0.0), (E, 0.0))
            return
        if steps == ["fn:tuple_uniform_encode"]:
            tag = self.tag_of(single_col())
            self.require(tag, scalar=False, types=NUM)
            for e in range(width):
                self.add(f"{name}_{e}", _SlotReq(tag, e, RED_NUM), (V, 1000.0), (V, 1000.0))
            self.checks.append((_SlotReq(tag, ELEM_WHOLE, RED_LEN), 0, float(width)))
            return
        if steps == ["fn:gt_encode_df"]:
            if single_col() != "gt" or "GT" not in self.header.formats:
                raise PlanError("gt_encode_df needs the FORMAT/GT tag")
            self.add(name, _SlotReq("GT", ELEM_WHOLE, RED_GT_HOM), (V, 0.0), (V, 0.0))
            return
        if steps == ["fn:allele_encode_df"]:
            if single_col() != "alleles":
                raise PlanError("allele_encode_df is only lowered for the alleles column")
            self.add(f"{name}_0", _SlotReq(None, 0, RED_FIX_ALLELE0), (V, 0.0), (V, 0.0))
            self.add(f"{name}_1", _SlotReq(None, 0, RED_FIX_ALLELE1), (E, 0.0), (E, 0.0))
            return
        if steps in (["fn:motif_encode_left_df"], ["fn:motif_encode_right_df"]):
            tag = self.tag_of(single_col())
            self.require(tag, scalar=None, types=(KIND_STR,))
            red = RED_MOTIF_L if "left" in steps[0] else RED_MOTIF_R
            self.add(name, _SlotReq(tag, ELEM_WHOLE, red), (E, 0.0), (E, 0.0))
            return
        if len(steps) == 2 and steps[0] == "impute:none:'FALSE'" and steps[1] == "ordinal":  # noqa: PLR2004
            tag = self.tag_of(single_col())
            self.require(tag, scalar=True, types=(KIND_STR,))
            if not hasattr(trans.steps[-1][1], "categories_"):
                raise PlanError(f"entry {name!r}: the OrdinalEncoder is not fitted")
            cats = list(trans.steps[-1][1].categories_[0])
            did = self.add_dict(cats)
            absent = (V, float(cats.index("FALSE"))) if "FALSE" in cats else (E, 0.0)
            self.add(name, _SlotReq(tag, 0, RED_DICT, did), absent, (E, 0.0))
            return
        if len(steps) == 2 and steps[0] == "impute:none:'0'" and steps[1] == "fn:convert_to_numeric":  # noqa: PLR2004
            tag = self.tag_of(single_col())
            self.require(tag, scalar=True, types=(KIND_STR, KIND_INT, KIND_FLOAT))
            is_str = all((k & 7) == KIND_STR for k in self._all_kinds(tag))
            if is_str:
                self.add(name, _SlotReq(tag, ELEM_WHOLE, RED_STRNUM), (V, 0.0), (E, 0.0))
            else:
                self.add(name, _SlotReq(tag, 0, RED_NUM), (V, 0.0), (V, 0.0))
            return
        # ---- CNV flavour (transformers.py:291-313)
        if steps == ["fn:svtype_encode_df"]:
            tag = self.tag_of(single_col())
            self.require(tag, scalar=True, types=(KIND_STR,))
            did = self.add_dict(["NEUTRAL", "DEL", "DUP"])  # index == svtype_encode code (transformers.py:80-83)
            self.add(name, _SlotReq(tag, 0, RED_DICT, did), (E, 0.0), (E, 0.0))
            return
        if steps == ["fn:copy_number_encode_df"]:
            if len(col_list) != 2:  # noqa: PLR2004
                raise PlanError(f"entry {name!r}: copy_number_encode_df takes two columns")
            tags = [self.tag_of(c) for c in col_list]
            for tag in tags:
                self.require(tag, scalar=True, types=NUM)
            n = POL_NULL
            self.add(name, _SlotReq(tags[0], 0, RED_NUM), (n, 0.0), (n, 0.0))
            self.combines.append((len(self.features) - 1, _SlotReq(tags[1], 0, RED_NUM)))
            return
        if steps == ["fn:cnv_source_encode_df"]:
            tag = self.tag_of(single_col())
            self.require(tag, scalar=False, types=(KIND_STR,))
            # index == cnv_source_encode code; index 0 is a string no VCF value can equal
            did = self.add_dict(["\x01", "cn.mops", "cnvpytor"])
            self.add(name, _SlotReq(tag, 0, RED_DICT, did), (E, 0.0), (E, 0.0))
            self.checks.append((_SlotReq(tag, ELEM_WHOLE, RED_LEN), 0, 1.0))  # len(x) != 1 -> ValueError
            self.checks.append((_SlotReq(tag, ELEM_WHOLE, RED_LEN), 1, 1.0))
            return
        if steps == ["fn:region_annotation_encode_df"]:
            from variantcalling_b200 import transformers as T

            tag = self.tag_of(single_col())
            self.require(tag, scalar=False, types=(KIND_STR,))
            names = sorted(T._REGIONS)  # noqa: SLF001
            lut = [1, 2, 3, 5, 4, 6, 7, 8]  # K1's table: subset bit mask (sorted names) -> code
            enc = T._get_region_encoding()  # noqa: SLF001
            for mask in range(8):
                subset = tuple(nm for i, nm in enumerate(names) if mask >> i & 1)
                if enc[subset] != lut[mask]:
                    raise PlanError("region encoding differs from the table compiled into K1")
            did = self.add_dict(names)
            self.add(name, _SlotReq(tag, ELEM_WHOLE, RED_REGION, did), (V, 0.0), (E, 0.0))
            return
        raise PlanError(f"entry {name!r}: transformer {steps} is not lowered by this build")


# --------------------------------------------------------------------------- models
def _f32_floor(t: np.ndarray) -> np.ndarray:
    """Largest float32 <= t (so ``x32 <= t64`` == ``x32 <= floor32(t64)``)."""
    t = np.asarray(t, dtype=np.float64)
    f = t.astype(np.float32)
    too_big = f.astype(np.float64) > t
    f[too_big] = np.nextafter(f[too_big], np.float32(-np.inf))
    return f


def _preorder_tree(left, right, feature, thr32, leaf_row_of, node_kind=None):
    """Child arrays (-1 = leaf) -> preorder node list [(is_leaf, thr | leaf_row, feature, right_rel, flags, cat_ref)].
    ``node_kind(n)`` -> (NODE_* flags, category bitset reference or None) of an internal node (default: (0, None))."""
    order, seq, stack = {}, [], [0]
    while stack:  # iterative DFS, left subtree first => left child is always the next node
        n = stack.pop()
        order[n] = len(seq)
        seq.append(n)
        if left[n] != -1:
            stack.append(int(right[n]))
            stack.append(int(left[n]))
    if len(seq) >= 65536:  # noqa: PLR2004
        raise PlanError("tree with more than 65535 nodes")
    nodes = []
    for n in seq:
        if left[n] == -1:
            nodes.append((True, int(leaf_row_of(n)), -1, 0, 0, None))
        else:
            if order[int(left[n])] != order[n] + 1:
                raise PlanError("internal error: preorder layout violated")
            flags, cat_ref = node_kind(n) if node_kind is not None else (0, None)
            nodes.append((False, float(thr32[n]), int(feature[n]), order[int(right[n])], flags, cat_ref))
    return nodes


def _pack_forest(trees, tree_out, leaves, leaf_width, cat_words=()) -> tuple[bytes, int, int]:
    """Forest section (plan.h): roots, tree outputs, preorder nodes, leaves, node flags, category bitset words."""
    roots = [0]
    node_bytes = bytearray()
    flags = bytearray()
    for nodes in trees:
        for is_leaf, value, feat, right, fl, cat_ref in nodes:
            if is_leaf:
                node_bytes += struct.pack("<ihH", value, -1, 0)
            elif cat_ref is not None:
                node_bytes += struct.pack("<IhH", cat_ref, feat, right)
            else:
                node_bytes += struct.pack("<fhH", value, feat, right)
            flags.append(fl)
        roots.append(roots[-1] + len(nodes))
    out = _pad8(np.asarray(roots, dtype="<u4").tobytes())
    out += _pad8(np.asarray(tree_out, dtype=np.uint8).tobytes())
    out += _pad8(bytes(node_bytes))
    out += _pad8(np.asarray(leaves, dtype="<f8").tobytes())
    out += _pad8(bytes(flags))
    out += struct.pack("<II", len(cat_words), sum(1 for f in flags if f))
    out += _pad8(np.asarray(cat_words, dtype="<u4").tobytes())
    return out, roots[-1], len(leaves) // max(1, leaf_width)


def _xgb_node_kinds(tr, ti: int, cat_words: list, bitset_at: dict):
    """-> node_kind(n) for _preorder_tree: the default-left / categorical flags of one xgboost tree, its category sets
    appended to ``cat_words`` as bitsets (bit c of word c // 32), each distinct bitset once (``bitset_at``: words ->
    first word).  A malformed category section raises PlanError."""
    n_nodes = len(tr["left_children"])
    split_type = np.asarray(tr.get("split_type") or [0] * n_nodes, dtype=np.int64)
    default_left = np.asarray(tr.get("default_left") or [0] * n_nodes, dtype=np.int64)
    if split_type.size != n_nodes or default_left.size != n_nodes:
        raise PlanError(f"xgboost tree {ti}: split_type / default_left do not have one entry per node")
    if ((split_type != 0) & (split_type != 1)).any():
        raise PlanError(f"xgboost tree {ti}: unknown split_type (0 numeric, 1 categorical)")
    cats = [int(c) for c in tr.get("categories", [])]
    c_nodes = [int(c) for c in tr.get("categories_nodes", [])]
    c_seg = [int(c) for c in tr.get("categories_segments", [])]
    c_size = [int(c) for c in tr.get("categories_sizes", [])]
    if not len(c_nodes) == len(c_seg) == len(c_size):
        raise PlanError(f"xgboost tree {ti}: categories_nodes / _segments / _sizes differ in length")
    ref_of = {}
    for nid, seg, size in zip(c_nodes, c_seg, c_size):
        if not 0 <= nid < n_nodes or split_type[nid] != 1:
            raise PlanError(f"xgboost tree {ti}: categories_nodes names node {nid}, which is not a categorical split")
        if seg < 0 or size < 1 or seg + size > len(cats):
            raise PlanError(f"xgboost tree {ti}: category segment [{seg}, {seg}+{size}) of node {nid} is out of range "
                            f"({len(cats)} categories)")
        codes = cats[seg:seg + size]
        if min(codes) < 0:
            raise PlanError(f"xgboost tree {ti}: node {nid} has a negative category code")
        if max(codes) >= MAX_CATEGORIES:
            raise PlanError(f"xgboost tree {ti}: node {nid} has category code {max(codes)}; codes must be below "
                            f"{MAX_CATEGORIES} (the category limit of the plan)")
        words = [0] * (max(codes) // 32 + 1)
        for c in codes:
            words[c // 32] |= 1 << (c % 32)
        key = tuple(words)
        if key not in bitset_at:
            if len(cat_words) + len(words) >= 1 << 24:
                raise PlanError("too many category bitset words")
            bitset_at[key] = len(cat_words)
            cat_words.extend(words)
        ref_of[nid] = bitset_at[key] | (len(words) << 24)
    left = tr["left_children"]
    for nid in range(n_nodes):
        if split_type[nid] == 1 and left[nid] != -1 and nid not in ref_of:
            raise PlanError(f"xgboost tree {ti}: categorical node {nid} is missing from categories_nodes")

    def node_kind(n):
        fl = (NODE_DEFAULT_LEFT if default_left[n] else 0) | (NODE_CATEGORICAL if split_type[n] == 1 else 0)
        return fl, ref_of.get(n)

    return node_kind


def _lower_model(model, n_features: int) -> dict:  # noqa: C901, PLR0912, PLR0915
    """-> dict(kind, n_classes, n_outputs, init[4], cmp, section bytes, n_trees, n_nodes, n_leaf_rows, leaf_width)."""
    init = [0.0] * MAX_CLASSES
    if isinstance(model, dict) or isinstance(model, (str, bytes)):
        return _lower_xgboost_json(model, n_features)
    cls = type(model).__name__
    if cls == "XGBClassifier":  # only reachable where xgboost is installed
        raw = model.get_booster().save_raw("json")
        return _lower_xgboost_json(json.loads(bytes(raw).decode()), n_features)
    if cls == "LogisticRegression":
        coef = np.asarray(model.coef_, dtype=np.float64)
        icpt = np.asarray(model.intercept_, dtype=np.float64)
        k = len(model.classes_)
        if coef.shape[1] != n_features:
            raise PlanError(f"model expects {coef.shape[1]} features, transformer yields {n_features}")
        n_out = coef.shape[0]
        if not ((k == 2 and n_out == 1) or (k > 2 and n_out == k)):  # noqa: PLR2004
            raise PlanError("unexpected LogisticRegression coefficient shape")
        if k > MAX_CLASSES:
            raise PlanError("too many classes")
        section = _pad8(coef.astype("<f8").tobytes()) + _pad8(icpt.astype("<f8").tobytes())
        return dict(kind=MODEL_LOGISTIC, n_classes=k, n_outputs=n_out, init=init, cmp=CMP_LE, section=section,
                    n_trees=0, n_nodes=0, n_leaf_rows=0, leaf_width=0, classes=list(model.classes_))
    if cls == "GradientBoostingClassifier":
        k = len(model.classes_)
        if k > MAX_CLASSES:
            raise PlanError("too many classes")
        est = model.estimators_
        n_out = est.shape[1]
        if getattr(model, "n_features_in_", n_features) != n_features:
            raise PlanError(f"model expects {model.n_features_in_} features, transformer yields {n_features}")
        raw0 = np.asarray(model._raw_predict_init(np.zeros((1, n_features))), dtype=np.float64).reshape(-1)  # noqa: SLF001
        for o in range(n_out):
            init[o] = float(raw0[o])
        scale = np.float64(model.learning_rate)
        trees, tree_out, leaves = [], [], []
        for stage in range(est.shape[0]):
            for o in range(n_out):
                t = est[stage, o].tree_
                base = len(leaves)
                leaf_ids = {}

                def leaf_row(n, t=t, base=base, leaf_ids=leaf_ids):
                    if n not in leaf_ids:
                        leaf_ids[n] = base + len(leaf_ids)
                        leaves.append(float(scale * np.float64(t.value[n, 0, 0])))
                    return leaf_ids[n]

                trees.append(_preorder_tree(t.children_left, t.children_right, t.feature,
                                            _f32_floor(t.threshold), leaf_row))
                tree_out.append(o)
        section, n_nodes, n_rows = _pack_forest(trees, tree_out, leaves, 1)
        return dict(kind=MODEL_GB_SKLEARN, n_classes=k, n_outputs=n_out, init=init, cmp=CMP_LE, section=section,
                    n_trees=len(trees), n_nodes=n_nodes, n_leaf_rows=n_rows, leaf_width=1,
                    classes=list(model.classes_))
    if cls == "RandomForestClassifier":
        k = len(model.classes_)
        if k > MAX_CLASSES:
            raise PlanError("too many classes")
        if getattr(model, "n_outputs_", 1) != 1:
            raise PlanError("multi-output forests are not lowered")
        trees, leaves = [], []
        for e in model.estimators_:
            t = e.tree_
            base = len(leaves) // k
            leaf_ids = {}

            def leaf_row(n, t=t, base=base, leaf_ids=leaf_ids):
                if n not in leaf_ids:
                    leaf_ids[n] = base + len(leaf_ids)
                    # DecisionTreeClassifier.predict_proba: value[:, :k] / row sum (0 -> 1)
                    v = np.asarray(t.value[n, 0, :k], dtype=np.float64).copy()
                    norm = v.sum()
                    if norm == 0.0:
                        norm = 1.0
                    leaves.extend((v / norm).tolist())
                return leaf_ids[n]

            trees.append(_preorder_tree(t.children_left, t.children_right, t.feature,
                                        _f32_floor(t.threshold), leaf_row))
        section, n_nodes, n_rows = _pack_forest(trees, [0] * len(trees), leaves, k)
        return dict(kind=MODEL_RF_SKLEARN, n_classes=k, n_outputs=k, init=init, cmp=CMP_LE, section=section,
                    n_trees=len(trees), n_nodes=n_nodes, n_leaf_rows=n_rows, leaf_width=k,
                    classes=list(model.classes_))
    raise PlanError(f"model type {cls} is not lowered (sklearn LogisticRegression / GradientBoostingClassifier / "
                    f"RandomForestClassifier, or an xgboost JSON dump)")


def _lower_xgboost_json(doc, n_features: int) -> dict:
    """xgboost >= 1.x ``Booster.save_model('*.json')`` document (gbtree, binary:logistic or
    multi:softprob).  PARITY UNPINNED: xgboost is not installed in the build container; the
    algorithm restated is xgboost 2.1.2's CPU predictor (fp32 ``x < split_condition`` goes
    left, fp32 margin accumulated in tree order from logit(base_score), fp32 sigmoid/softmax),
    with its missing-value and categorical routing (``GetNextNode`` / ``common::Decision``): NaN
    takes the node's default child (``default_left``); a categorical node (``split_type`` 1, its set
    in ``categories[categories_segments[i]:][:categories_sizes[i]]``) sends a category in the set
    right and everything else (not in the set, negative, >= 2^24) left.  Category codes must be
    below ``MAX_CATEGORIES``."""
    if isinstance(doc, (str, bytes)):
        try:
            doc = json.loads(doc)
        except (UnicodeDecodeError, json.JSONDecodeError):
            if isinstance(doc, str):
                raise
            from variantcalling_b200 import ubjson  # the binary flavour (save_model("*.ubj"), save_raw("ubj"))

            doc = ubjson.loads(doc)
    learner = doc["learner"]
    objective = learner["objective"]["name"]
    lmp = learner["learner_model_param"]
    num_class = int(lmp.get("num_class", "0"))
    base_score = np.float32(float(lmp.get("base_score", "0.5")))
    gb = learner["gradient_booster"]
    if gb.get("name", "gbtree") != "gbtree":
        raise PlanError("only the gbtree booster is lowered")
    model = gb["model"]
    tree_info = model["tree_info"]
    init = [0.0] * MAX_CLASSES
    if objective == "binary:logistic":
        k, n_out = 2, 1
        init[0] = float(np.float32(-np.log(np.float32(1.0) / base_score - np.float32(1.0))))
    elif objective in ("multi:softprob", "multi:softmax"):
        k = n_out = num_class
        if k > MAX_CLASSES:
            raise PlanError("too many classes")
        for o in range(k):
            init[o] = float(base_score)
    else:
        raise PlanError(f"xgboost objective {objective} is not lowered")
    trees, tree_out, leaves, cat_words, bitset_at = [], [], [], [], {}
    for ti, tr in enumerate(model["trees"]):
        node_kind = _xgb_node_kinds(tr, ti, cat_words, bitset_at)
        left = np.asarray(tr["left_children"], dtype=np.int64)
        right = np.asarray(tr["right_children"], dtype=np.int64)
        feat = np.asarray(tr["split_indices"], dtype=np.int64)
        cond = np.asarray(tr["split_conditions"], dtype=np.float32)
        if feat.size and feat.max() >= n_features:
            raise PlanError("xgboost split index beyond the transformer's feature count")
        base = len(leaves)
        leaf_ids = {}

        def leaf_row(n, cond=cond, base=base, leaf_ids=leaf_ids):
            if n not in leaf_ids:
                leaf_ids[n] = base + len(leaf_ids)
                leaves.append(float(cond[n]))
            return leaf_ids[n]

        trees.append(_preorder_tree(left, right, feat, cond, leaf_row, node_kind))
        tree_out.append(int(tree_info[ti]) if n_out > 1 else 0)
    section, n_nodes, n_rows = _pack_forest(trees, tree_out, leaves, 1, cat_words)
    return dict(kind=MODEL_XGB, n_classes=k, n_outputs=n_out, init=init, cmp=CMP_LT, section=section,
                n_trees=len(trees), n_nodes=n_nodes, n_leaf_rows=n_rows, leaf_width=1, classes=list(range(k)))


# --------------------------------------------------------------------------- entry point
def compile_plan(header: VcfHeader | str | bytes, transformer, model, custom_info_fields=None) -> Plan:  # noqa: C901
    """Lower a fitted (transformer, model) pair against a VCF header."""
    if not isinstance(header, VcfHeader):
        header = VcfHeader(header)
    b = _Builder(header, custom_info_fields)
    if not hasattr(transformer, "transformers_"):
        raise PlanError("the transformer is not fitted (no transformers_ attribute)")
    out_idx = getattr(transformer, "output_indices_", {})
    for name, trans, cols in transformer.transformers_:
        if name == "remainder":
            if trans != "drop":
                raise PlanError("remainder='passthrough' is not lowered")
            continue
        sl = out_idx.get(name)
        width = (sl.stop - sl.start) if sl is not None else 1
        before = len(b.features)
        b.lower_entry(name, trans, cols, width)
        if sl is not None and len(b.features) - before != width:
            raise PlanError(f"entry {name!r}: fitted width {width} != lowered width {len(b.features) - before}")
    n_feat = len(b.features)
    if n_feat == 0 or n_feat > MAX_FEATURES:
        raise PlanError(f"feature count {n_feat} out of range")
    m = _lower_model(model, n_feat)

    # ---- slot layout: per-tag contiguous, fixed-column slots last
    reqs: list[_SlotReq] = [f.slot for f in b.features] + [c[0] for c in b.checks] + [c[1] for c in b.combines]
    tag_names = []
    for r in reqs:
        if r.tag is not None and r.tag not in tag_names:
            tag_names.append(r.tag)
    if len(tag_names) > MAX_TAGS:
        raise PlanError("too many tags")
    slot_index: dict[tuple, int] = {}
    slots: list[tuple] = []
    tags_packed = []
    for ti, tag in enumerate(tag_names):
        if len(tag.encode()) > NAME_MAX:
            raise PlanError(f"tag name {tag!r} longer than {NAME_MAX} bytes")
        first = len(slots)
        # K1 contract: element slots 0..k-1 (each element once, gaps filled with unused numeric
        # slots), then at most one whole-value slot
        by_elem: dict[int, _SlotReq] = {}
        whole_req = None
        for r in reqs:
            if r.tag != tag:
                continue
            if r.elem == ELEM_WHOLE:
                if whole_req is not None and (whole_req.reducer, whole_req.dict_id) != (r.reducer, r.dict_id):
                    raise PlanError(f"tag {tag}: more than one whole-value reducer")
                whole_req = r
            else:
                prev = by_elem.get(r.elem)
                if prev is not None and (prev.reducer, prev.dict_id) != (r.reducer, r.dict_id):
                    raise PlanError(f"tag {tag}: element {r.elem} is reduced in two different ways")
                by_elem[r.elem] = r
        for e in range(max(by_elem) + 1 if by_elem else 0):
            r = by_elem.get(e) or _SlotReq(tag, e, RED_NUM)
            slot_index[(tag, e, r.reducer, r.dict_id)] = len(slots)
            slots.append((ti, e, r.reducer, r.dict_id))
        if whole_req is not None:
            slot_index[(tag, ELEM_WHOLE, whole_req.reducer, whole_req.dict_id)] = len(slots)
            slots.append((ti, ELEM_WHOLE, whole_req.reducer, whole_req.dict_id))
        ik, fk = b.kinds(tag)
        name_b = tag.encode()
        whole_red, whole_slot = (whole_req.reducer, len(slots) - 1) if whole_req is not None else (0xFF, 0)
        tags_packed.append(struct.pack("<32sBBBBBBBx", name_b, len(name_b), ik, fk, first, len(slots) - first,
                                       whole_red, whole_slot))
    for r in reqs:
        key = (r.tag, r.elem, r.reducer, r.dict_id)
        if r.tag is None and key not in slot_index:
            slot_index[key] = len(slots)
            slots.append((TAG_FIXED, r.elem, r.reducer, r.dict_id))
    if len(slots) > MAX_SLOTS:
        raise PlanError("too many raw slots")

    def sid(r: _SlotReq) -> int:
        return slot_index[(r.tag, r.elem, r.reducer, r.dict_id)]

    if len(b.dicts) > MAX_DICTS or sum(len(d) for d in b.dicts) > MAX_STRINGS:
        raise PlanError("too many OrdinalEncoder categories for the K1 dictionary tables")
    strings = []
    dicts_packed = b""
    for d in b.dicts:
        dicts_packed += struct.pack("<HH", len(strings), len(d))
        strings.extend(d)
    strings_packed = b"".join(struct.pack("<24sB7x", s.encode(), len(s.encode())) for s in strings)
    feats_packed = b"".join(
        struct.pack("<HBBff", sid(f.slot), f.absent[0], f.missing[0], f.absent[1], f.missing[1]) for f in b.features)
    checks_packed = b"".join(struct.pack("<HBxf", sid(c[0]), c[1], c[2]) for c in b.checks)
    combines_packed = b"".join(struct.pack("<HHB3x", c[0], sid(c[1]), 0) for c in b.combines)
    hdr = struct.pack(
        "<15I2H4d", PLAN_MAGIC, PLAN_VERSION, len(tags_packed), len(slots), n_feat, len(b.dicts), len(strings),
        m["kind"], m["n_classes"], m["n_outputs"], m["n_trees"], m["n_nodes"], m["n_leaf_rows"], m["leaf_width"],
        m["cmp"], len(b.checks), len(b.combines), *m["init"])
    blob = (_pad8(hdr) + _pad8(b"".join(tags_packed)) + _pad8(b"".join(struct.pack("<4B", *s) for s in slots))
            + _pad8(dicts_packed) + _pad8(strings_packed) + _pad8(feats_packed) + _pad8(checks_packed)
            + _pad8(combines_packed) + m["section"])
    return Plan(blob=blob, n_features=n_feat, n_classes=m["n_classes"], n_slots=len(slots), tags=tag_names,
                feature_names=b.feature_names, model_kind=m["kind"], classes=m.get("classes", []))


def compile_plan_model_only(model, n_features: int) -> Plan:
    """Plan that carries only the model (for ``ugvc_predict_features``: K3 on a dense feature matrix the
    caller assembled itself, e.g. ``variant_filtering_utils.apply_model`` with the transformer on the host).
    The feature table is a placeholder (one fixed slot) -- K1 / K2 never run on this plan."""
    if n_features < 1 or n_features > MAX_FEATURES:
        raise PlanError(f"feature count {n_features} out of range")
    m = _lower_model(model, n_features)
    slots = [(TAG_FIXED, 0, RED_FIX_QUAL, 0)]
    feats_packed = b"".join(struct.pack("<HBBff", 0, POL_NULL, POL_NULL, 0.0, 0.0) for _ in range(n_features))
    hdr = struct.pack("<15I2H4d", PLAN_MAGIC, PLAN_VERSION, 0, len(slots), n_features, 0, 0, m["kind"], m["n_classes"],
                      m["n_outputs"], m["n_trees"], m["n_nodes"], m["n_leaf_rows"], m["leaf_width"], m["cmp"], 0, 0,
                      *m["init"])
    blob = (_pad8(hdr) + _pad8(b"") + _pad8(b"".join(struct.pack("<4B", *x) for x in slots)) + _pad8(b"") + _pad8(b"")
            + _pad8(feats_packed) + _pad8(b"") + _pad8(b"") + m["section"])
    return Plan(blob=blob, n_features=n_features, n_classes=m["n_classes"], n_slots=len(slots), tags=[],
                feature_names=[f"x{i}" for i in range(n_features)], model_kind=m["kind"], classes=m.get("classes", []))


def compile_plan_no_model(header: VcfHeader | str | bytes) -> Plan:
    """Plan for runs without ``--model_file``: only K0/K1 run (line index, POS, column
    offsets, CG flag) so the writer can apply the blacklist / PASS-fill rules."""
    if not isinstance(header, VcfHeader):
        header = VcfHeader(header)
    hdr = struct.pack("<15I2H4d", PLAN_MAGIC, PLAN_VERSION, 0, 0, 0, 0, 0, 0, 2, 1, 0, 0, 0, 0, CMP_LE, 0, 0,
                      0.0, 0.0, 0.0, 0.0)
    return Plan(blob=_pad8(hdr), n_features=0, n_classes=2, n_slots=0, tags=[], feature_names=[], model_kind=0)
