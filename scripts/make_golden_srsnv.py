#!/usr/bin/env python
"""Generate tests/golden/srsnv_kfold.npz from the REFERENCE's own srsnv k-fold model step (run where the reference
sources are; the fixture travels, the reference does not).

``ugbio_srsnv.srsnv_training_utils`` imports pysam, xgboost, simppl, matplotlib, the featuremap / ppmSeq helpers and
the srsnv plotting module at the top; neither of the two functions used here needs them, so they are replaced by
empty stand-in modules.  Everything exercised is the unmodified reference code: ``set_categorical_columns`` and ``k_fold_predict_proba`` (with ``return_train=False``, what
``MLQualAnnotator.process_records`` calls).  The models are the reference's two srsnv fold models
(tests/golden/416119_L7402.test.model_fold_{0,1}.json.gz) evaluated by the restated xgboost predictor
(tests/xgb_categorical_ref.py) behind a ``predict_proba`` that returns float32, as XGBClassifier's does.

The frame (seeded): the model's 26 features, categorical values drawn from the metadata's category maps plus unknown
ones (they become NaN codes), NaN numerics, and a fold column with valid folds (0, 1), NaN (no fold: the mean phred
over both models) and out-of-range folds (-1, 2, 5: NaN out).

Harness shim: the reference starts ``preds`` as ``pd.Series(0, ...)`` (int64) and assigns float probabilities into
it, which pandas 3 refuses; ``pd.Series`` called with exactly ``(0, index=..., name="test")`` is given a float64 0.0
instead (the same values: 0 + x is x either way).

Output: srsnv_kfold.npz with the frame's feature matrix as xgboost reads it (float32, category codes, NaN), the fold
column (float64, NaN for none) and the reference's predictions (float64).
"""
import gzip
import json
import os
import sys
import types

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = "/root/reference/ugbio_utils/src"
for sub in ("srsnv", "core"):
    sys.path.insert(0, os.path.join(REF, sub))


class _Anything:
    """Stand-in for every name the import-only modules provide (module-level constants reach through it)."""

    def __getattr__(self, name):
        return _Anything()

    def __call__(self, *a, **k):
        return _Anything()


def _stub(name):
    mod = types.ModuleType(name)
    mod.__getattr__ = lambda attr: _Anything()
    sys.modules[name] = mod


for name in ("pysam", "xgboost", "simppl", "simppl.simple_pipeline", "ugbio_srsnv.srsnv_plotting_utils", "matplotlib",
             "matplotlib.pyplot", "ugbio_featuremap", "ugbio_featuremap.featuremap_utils", "ugbio_ppmseq",
             "ugbio_ppmseq.ppmSeq_utils"):
    _stub(name)

_Series = pd.Series


class _HarnessSeries(_Series):  # pandas-3 harness shim (see the module docstring)
    def __init__(self, data=None, *args, **kwargs):
        if isinstance(data, int) and data == 0 and kwargs.get("name") == "test" and not args:
            data = 0.0
        super().__init__(data, *args, **kwargs)


from ugbio_srsnv import srsnv_training_utils as T  # noqa: E402

T.pd = types.SimpleNamespace(**{k: getattr(pd, k) for k in dir(pd) if not k.startswith("__")})
T.pd.Series = _HarnessSeries

from tests import xgb_categorical_ref as XR  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def main():
    features = XR.metadata_features()
    docs = [json.load(gzip.open(os.path.join(GOLDEN, f"416119_L7402.test.model_fold_{k}.json.gz"))) for k in (0, 1)]
    names = docs[0]["learner"]["feature_names"]
    assert [f["name"] for f in features] == names
    n = 4000
    df = XR.srsnv_frame(2024, n, features)
    cat_dict = {f["name"]: list(f["values"]) for f in features if f["type"] == "c"}
    df = T.set_categorical_columns(df, cat_dict)
    fold = XR.srsnv_folds(7, n)
    df["fold_id"] = fold
    models = [XR.OracleModel(d) for d in docs]
    preds = T.k_fold_predict_proba(models, df, names, 2, kfold_col="fold_id", return_train=False)
    from variantcalling_b200 import model_apply as MA

    np.savez_compressed(os.path.join(GOLDEN, "srsnv_kfold.npz"), x=MA.frame_matrix(df[names], names),
                        fold=fold.astype(np.float64), preds=preds.to_numpy(dtype=np.float64))
    print(f"srsnv_kfold.npz: {n} rows, {int(np.isnan(preds).sum())} NaN predictions")


if __name__ == "__main__":
    main()
