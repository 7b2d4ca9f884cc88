"""The model-apply step on its own: ``predict_proba`` / ``predict`` of a fitted model on the GPU (K3).

``apply_model(input_df, model, transformer)`` mirrors
``ugbio_filtering/variant_filtering_utils.py:95-125`` (transform in chunks on the host, null check,
then the model -- here one K3 launch per chunk instead of ``model.predict`` + ``model.predict_proba``),
and :class:`GpuClassifier` gives the same step to the other model-apply tools the reference has
(``featuremap_xgb_prediction.predict_record_with_xgb``, ``srsnv_inference_utils``: a feature frame and
an xgboost / sklearn classifier).  Supported models: what ``model_compiler`` lowers (sklearn
LogisticRegression / GradientBoostingClassifier / RandomForestClassifier, xgboost JSON or Booster).
Probabilities come back in the trainer's precision (fp64 for sklearn, fp32 values for xgboost).
``GpuClassifier.predict_proba`` takes a matrix or a data frame; a frame is read the way xgboost's DMatrix reads one
with ``enable_categorical`` (category columns become their codes, an unknown category NaN).  For an xgboost model NaN
is a missing value, routed to each node's default child; sklearn models refuse it as sklearn does.
``k_fold_predict_proba`` and ``ml_qual`` are the model step of the srsnv inference
(``ugbio_srsnv/srsnv_training_utils.py:222-290``, ``srsnv_inference_utils.py:163-211``).
``predict_record_with_xgb`` is the model step of the featuremap tool
(``ugbio_featuremap/featuremap_xgb_prediction.py:258-262,301-323``) with the same signature: the frame its
``df_vcf_manual_aggregation`` built, the model file, the probability of class 1 back.
There is no CPU path.
"""
from __future__ import annotations

import json

import numpy as np
import pandas as pd

from variantcalling_b200 import lib
from variantcalling_b200 import model_compiler as MC

MAX_CHUNK_SIZE = 1000000  # variant_filtering_utils.py:18


class GpuClassifier:
    def __init__(self, model, n_features: int | None = None, device: int = 0, max_rows: int = 1 << 20):
        if n_features is None:
            n_features = getattr(model, "n_features_in_", None)
        if n_features is None:
            raise ValueError("n_features is needed for a model that does not record n_features_in_")
        self.plan = MC.compile_plan_model_only(model, int(n_features))
        self.feature_names = None  # an xgboost document's feature_names: a frame's columns must match them
        if isinstance(model, (dict, str, bytes)):  # a document, or its JSON / UBJSON text as the compiler takes it
            doc = load_xgb_document(model.encode() if isinstance(model, str) else model)
            self.feature_names = doc["learner"].get("feature_names") or None
        self.classes_ = np.asarray(self.plan.classes if len(self.plan.classes) else np.arange(self.plan.n_classes))
        self.ctx = lib.Context(device)
        self.ctx.load_plan(self.plan.blob)
        self.ctx.enable_phreds(2)  # K3 keeps the fp64 class probabilities
        self.max_rows = 0
        self._reserve(max_rows)

    def _reserve(self, rows: int):
        if rows > self.max_rows:
            self.max_rows = int(rows)
            self.ctx.reserve(4096, self.max_rows, 1)

    def close(self):
        self.ctx.close()

    def predict_proba(self, x) -> np.ndarray:
        if isinstance(x, pd.DataFrame):
            x = frame_matrix(x, self.feature_names)
        x = x.to_numpy() if hasattr(x, "to_numpy") else np.asarray(x)
        if x.ndim != 2 or x.shape[1] != self.plan.n_features:
            raise ValueError(f"X has {x.shape[1] if x.ndim == 2 else '?'} features, the model expects {self.plan.n_features}")
        if self.plan.model_kind == MC.MODEL_XGB:  # NaN is xgboost's missing value
            if np.isinf(np.asarray(x, dtype=np.float64)).any():
                raise ValueError("Input X contains infinity")
        elif not np.isfinite(np.asarray(x, dtype=np.float64)).all():
            raise ValueError("Input X contains NaN or infinity")  # sklearn's check_array message, in short
        out = np.empty((x.shape[0], self.plan.n_classes), dtype=np.float64)
        step = min(self.max_rows, MAX_CHUNK_SIZE)
        for b in range(0, x.shape[0], step):
            part = np.ascontiguousarray(x[b:b + step], dtype=np.float32)
            self.ctx.predict_features(part)
            out[b:b + part.shape[0]] = self.ctx.collect_phreds(0, part.shape[0])
        return out

    def predict(self, x) -> np.ndarray:
        return self.classes_[np.argmax(self.predict_proba(x), axis=1)]


def frame_matrix(df: pd.DataFrame, feature_names=None) -> np.ndarray:
    """A feature frame as xgboost's DMatrix reads it with ``enable_categorical``: a category column becomes its codes
    (-1, a value outside the categories or a missing one, becomes NaN), a numeric or boolean column float32 (nulls
    NaN).  Object / string columns are refused, as xgboost refuses them.  With ``feature_names`` (the model's) the
    columns must be exactly those, in that order."""
    if feature_names is not None and list(df.columns) != list(feature_names):
        raise ValueError(f"feature_names mismatch: the model expects {list(feature_names)}, the frame has {list(df.columns)}")
    out = np.empty((df.shape[0], df.shape[1]), dtype=np.float32)
    for i, name in enumerate(df.columns):
        col = df[name]
        if isinstance(col.dtype, pd.CategoricalDtype):
            codes = col.cat.codes.to_numpy()
            out[:, i] = np.where(codes < 0, np.nan, codes).astype(np.float32)
        elif pd.api.types.is_bool_dtype(col.dtype) or pd.api.types.is_numeric_dtype(col.dtype):
            out[:, i] = col.to_numpy(dtype=np.float64, na_value=np.nan).astype(np.float32)
        else:
            raise ValueError(f"column {name!r} has dtype {col.dtype}: only numeric, boolean and category columns are "
                             f"model features (make it categorical)")
    return out


def _validate_data(data) -> None:
    """variant_filtering_utils.py:128-143"""
    arr = data if isinstance(data, np.ndarray) else pd.DataFrame(data).to_numpy()
    if arr.ndim == 1 or arr.shape[1] <= 1:
        assert pd.isna(arr).sum() == 0, "data vector contains null"  # noqa: S101
    else:
        for c in range(arr.shape[1]):
            assert pd.isna(arr[:, c]).sum() == 0, f"Data matrix contains null in column {c}"  # noqa: S101


def apply_model(input_df: pd.DataFrame, model, transformer, classifier: GpuClassifier | None = None):
    """-> (predictions, probabilities) like variant_filtering_utils.apply_model (:95-125)."""
    chunks = np.arange(0, input_df.shape[0], MAX_CHUNK_SIZE, dtype=int)
    chunks = np.concatenate((chunks, [input_df.shape[0]]))
    parts = [transformer.transform(input_df.iloc[chunks[i]:chunks[i + 1]]) for i in range(len(chunks) - 1)]
    x_test = pd.concat(parts)
    _validate_data(x_test)
    own = classifier is None
    clf = classifier or GpuClassifier(model, n_features=x_test.shape[1], max_rows=min(MAX_CHUNK_SIZE, max(1, x_test.shape[0])))
    try:
        probabilities = clf.predict_proba(x_test)
        predictions = clf.classes_[np.argmax(probabilities, axis=1)]
    finally:
        if own:
            clf.close()
    return predictions, probabilities


# ------------------------------------------------------------------ featuremap_xgb_prediction.py:258-262,301-323
def set_categorial_columns(df: pd.DataFrame) -> None:
    """In place, like the reference's helper: every object / category column becomes the rank of ``str(value)`` among
    the sorted distinct strings of THIS frame (``LabelEncoder().fit_transform(df[col].astype(str))``)."""
    for col in df.select_dtypes(include=["object", "category", "string"]).columns:
        _, codes = np.unique(df[col].astype(str).to_numpy(dtype=object).astype(str), return_inverse=True)
        df[col] = codes.astype(np.int64)


def load_xgb_document(xgb_model) -> dict:
    """The model file of ``XGBClassifier.load_model`` (JSON or UBJSON), a parsed document, or raw bytes of either."""
    if isinstance(xgb_model, dict):
        return xgb_model
    raw = xgb_model
    if isinstance(xgb_model, str):
        with open(xgb_model, "rb") as fh:
            raw = fh.read()
    try:
        return json.loads(raw)
    except (UnicodeDecodeError, json.JSONDecodeError):
        from variantcalling_b200 import ubjson

        return ubjson.loads(bytes(raw))


def predict_record_with_xgb(df_variants: pd.DataFrame, xgb_model, classifier: GpuClassifier | None = None) -> np.ndarray:
    """-> probability of class "1" for every row (the reference's ``df_probabilities["1"].to_numpy()``).
    Columns = the booster's ``feature_names``; object columns label-encoded per call, nulls filled with 0; then K3."""
    doc = load_xgb_document(xgb_model)
    features = doc["learner"].get("feature_names") or []
    if not features:
        raise ValueError("the model document carries no feature_names (it was not trained on a data frame)")
    x = df_variants[list(features)].copy()
    set_categorial_columns(x)
    x = x.fillna(0)
    own = classifier is None
    clf = classifier or GpuClassifier(doc, n_features=len(features), max_rows=min(MAX_CHUNK_SIZE, max(1, x.shape[0])))
    try:
        if x.shape[0] == 0:
            return np.zeros(0, dtype=np.float32)
        probabilities = clf.predict_proba(x.to_numpy(dtype=np.float32))
    finally:
        if own:
            clf.close()
    return probabilities[:, 1].astype(np.float32)  # xgboost's probabilities are fp32 values


# ------------------------------------------------------------------ srsnv: srsnv_training_utils.py:204-290
FOLD_ID = "fold_id"


def prob_to_phred(prob, eps=1e-8):
    """srsnv_training_utils.py:204-211"""
    return -10 * np.log10(1 - prob + eps)


def phred_to_prob(phred):
    """srsnv_training_utils.py:214-219"""
    return 1.0 - 10.0 ** (-phred / 10)


def _class1(model, frame) -> np.ndarray:
    """Class-1 probability; float32 for an xgboost model, as its predict_proba returns it (prob_to_phred then computes
    in float32, as the reference does)."""
    p = model.predict_proba(frame)[:, 1]
    return p.astype(np.float32) if getattr(getattr(model, "plan", None), "model_kind", None) == MC.MODEL_XGB else p


def k_fold_predict_proba(models, df: pd.DataFrame, columns_for_training, k_folds: int, kfold_col: str = FOLD_ID) -> pd.Series:
    """The k-fold model step of srsnv inference (``srsnv_training_utils.k_fold_predict_proba`` with
    ``return_train=False``): a row whose fold is in [0, k_folds) gets the class-1 probability of its own fold's model;
    a row without a fold (NaN) gets the mean over all models of ``prob_to_phred(p)``, mapped back with
    ``phred_to_prob``; any other row is NaN.  ``models``: one :class:`GpuClassifier` per fold."""
    fold = df[kfold_col]
    test_cond = fold.isna().to_numpy()
    fold_v = fold.to_numpy(dtype=np.float64, na_value=np.nan)
    preds = np.zeros(df.shape[0], dtype=np.float64)
    all_val = test_cond.copy()
    cols = list(columns_for_training)
    for k in range(k_folds):
        val_cond = fold_v == k
        all_val |= val_cond
        if val_cond.any():
            preds[val_cond] = _class1(models[k], df.loc[val_cond, cols])
        if test_cond.any():
            preds[test_cond] += prob_to_phred(_class1(models[k], df.loc[test_cond, cols])) / k_folds
    preds[test_cond] = phred_to_prob(preds[test_cond])
    preds[~all_val] = np.nan
    return pd.Series(preds, index=df.index, name="test")


def set_categorical_columns(df: pd.DataFrame, cat_dict: dict) -> pd.DataFrame:
    """srsnv_training_utils.py:144-161: a copy whose columns named in ``cat_dict`` are categoricals over exactly those
    categories (a value outside them becomes a missing category)."""
    df = df.copy()
    for col, cats in cat_dict.items():
        known = df[col].isin(cats)  # the others become missing categories
        df[col] = df[col].where(known).astype(pd.CategoricalDtype(cats, ordered=False))
    return df


def ml_qual(models, variants_df: pd.DataFrame, categorical_features_dict: dict, numerical_features,
            chrom_folds: dict | None = None) -> np.ndarray:
    """The frame part of srsnv's ``MLQualAnnotator.process_records`` (``srsnv_inference_utils.py:163-211``, without
    the pre-filter and the quality interpolation): categoricals set, ``rq`` as float, the fold of each row from
    ``chrom_folds`` (by its ``chrom``; every row fold 0 with one model, no fold without ``chrom_folds``), the k-fold
    probability, and ML_QUAL = ``clip(-10 log10(1 - p), 0)`` for every row."""
    categorical = list(categorical_features_dict)
    df = set_categorical_columns(variants_df, categorical_features_dict)
    if "rq" in df.columns:
        df = df.astype({"rq": float})
    features = list(numerical_features) + categorical
    if len(models) == 1:
        df[FOLD_ID] = 0
    elif chrom_folds is None:
        df[FOLD_ID] = np.nan
    else:
        df[FOLD_ID] = df["chrom"].map(chrom_folds, na_action="ignore").astype("Int64")
    p = k_fold_predict_proba(models, df, features, len(models), kfold_col=FOLD_ID).to_numpy()
    with np.errstate(divide="ignore"):
        return (-10 * np.log10(1 - p)).clip(min=0)
