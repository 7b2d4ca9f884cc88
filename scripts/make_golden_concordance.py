#!/usr/bin/env python
"""Generate tests/golden/concordance_metrics.json.gz from the REFERENCE's own
``ugbio_core.concordance.concordance_utils`` (calc_accuracy_metrics, calc_recall_precision_curve)
imported from /root/reference -- they need only numpy / pandas / sklearn, all present here.

One harness note: the reference is pinned to pandas < 3, where ``pd.concat`` ignores the empty
``init_metrics_df()`` frame when it picks dtypes, so ``accuracy_df.round(5)`` rounds; pandas 3 keeps
``object`` columns and the round is a no-op.  The fixture stores what the functions return here
(unrounded); the tests round both sides to 5 decimals, the behaviour in the reference's own
environment.

Besides make_cases, the fixture holds make_edge_cases (score families and group edges) and make_error_cases (non-finite
scores): for each function either its output or, where it raises, {"error": [exception type, message]}.  "_meta" records
the scikit-learn version the curves came from.  Signed zeros are left out: scikit-learn >= 1.6 (a stable descending
sort) reports a tie run's last zero where the reference's pin (1.5.x, a stable ascending sort reversed) reports its
first, so the tests pin that rule with a known-answer table instead.
"""
import gzip
import json
import os
import sys
import warnings

import numpy as np
import pandas as pd
import sklearn

warnings.filterwarnings("ignore")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference/ugbio_utils/src/core")

from ugbio_core.concordance import concordance_utils as ref_cu  # noqa: E402

from tests.concordance_data import make_cases, make_edge_cases, make_error_cases  # noqa: E402


def jsonable(v):
    if isinstance(v, (list, tuple, np.ndarray)):
        return [jsonable(x) for x in v]
    if isinstance(v, (np.integer,)):
        return int(v)
    if isinstance(v, (float, np.floating)):
        return None if np.isnan(v) else float(v)
    return v


def frame_or_error(fn, *args):
    try:
        with pd.option_context("future.infer_string", False):
            res = fn(*args)
    except Exception as e:  # noqa: BLE001
        return {"error": [type(e).__name__, str(e)]}
    return {c: jsonable(list(res[c])) for c in res.columns}


def main():
    out = {"_meta": {"sklearn": sklearn.__version__}}
    for name, df, classify_col, group_col in [*make_cases(), *make_edge_cases(), *make_error_cases()]:
        out[name] = {
            "accuracy": frame_or_error(ref_cu.calc_accuracy_metrics, df.copy(), classify_col, None, group_col),
            "curve": frame_or_error(ref_cu.calc_recall_precision_curve, df.copy(), classify_col, None, group_col),
        }
        acc, curve = out[name]["accuracy"], out[name]["curve"]
        print(name, df.shape, "groups", acc.get("group", acc.get("error")),
              "curve points", [len(p) for p in curve["precision"]] if "precision" in curve else curve["error"])
    path = os.path.join(ROOT, "tests", "golden", "concordance_metrics.json.gz")
    with gzip.open(path, "wt", compresslevel=9) as fh:
        json.dump(out, fh)
    print("wrote", path, os.path.getsize(path) >> 10, "KiB")


if __name__ == "__main__":
    main()
