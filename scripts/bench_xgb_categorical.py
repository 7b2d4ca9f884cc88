#!/usr/bin/env python
"""K3 throughput on the srsnv fold-0 model (26 features, 20 trees of depth 10, 874 categorical nodes: k3_infer with
the categorical walk) beside the same forest with its categorical nodes made numeric (threshold = smallest code of
the set + 0.5, default-left kept: same walk, no bitset lookups) and with neither categorical nodes nor default-left
flags (the plain walk).

Rows are scored through ugvc_predict_features in batches; K3's time is the sum of the k3_* kernel durations
torch.profiler records (CUDA activities), so host staging and copies are not counted.  Prints one JSON line with the
card name and power limit (nvidia-smi) and K3 rows/s of each variant.

    python scripts/bench_xgb_categorical.py --rows 16777216 --batch 4194304
"""
import argparse
import copy
import gzip
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from variantcalling_b200 import lib  # noqa: E402
from variantcalling_b200 import model_compiler as MC  # noqa: E402


def _numeric(doc, keep_default_left: bool):
    doc = copy.deepcopy(doc)
    for tr in doc["learner"]["gradient_booster"]["model"]["trees"]:
        for nid, seg, size in zip(tr["categories_nodes"], tr["categories_segments"], tr["categories_sizes"]):
            tr["split_conditions"][nid] = float(min(tr["categories"][seg:seg + size])) + 0.5
        n = len(tr["left_children"])
        tr.update(split_type=[0] * n, categories=[], categories_nodes=[], categories_segments=[], categories_sizes=[])
        if not keep_default_left:
            tr["default_left"] = [0] * n
    return doc


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 24)
    ap.add_argument("--batch", type=int, default=1 << 22)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    with gzip.open(os.path.join(ROOT, "tests", "golden", "416119_L7402.test.model_fold_0.json.gz")) as fh:
        doc = json.load(fh)
    rng = np.random.default_rng(a.seed)
    x = np.empty((a.batch, 26), dtype=np.float32)
    x[:, :8] = rng.integers(0, 14, size=(a.batch, 8))                 # categorical columns: codes
    x[:, 8:] = np.round(rng.gamma(2.0, 20.0, size=(a.batch, 18)))
    x[:, [19, 21, 22]] = rng.integers(0, 14, size=(a.batch, 3))
    x[:, 20] = rng.random(a.batch)
    x[rng.random(x.shape) < 0.02] = np.nan
    out = {"model": "srsnv fold 0 (26 features, 20 trees, depth 10)", "rows": 0}
    out["gpu"], out["power_limit"] = _card()
    for label, d in (("categorical", doc), ("numeric_default_left", _numeric(doc, True)), ("plain", _numeric(doc, False))):
        ctx = lib.Context(0)
        ctx.load_plan(MC.compile_plan_model_only(d, 26).blob)
        ctx.reserve(4096, a.batch, 1)
        ctx.predict_features(x)  # warm-up
        torch.cuda.synchronize()
        n_batches = max(1, a.rows // a.batch)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_batches):
                ctx.predict_features(x)
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if e.key.startswith("void k3_") or e.key.startswith("k3_"))
        out[label] = {"walk": ctx.k3_config()["walk"], "kernel": ctx.k3_config()["kernel"],
                      "k3_ms": round(us / 1000.0, 3), "k3_rows_per_s": round(n_batches * a.batch / (us * 1e-6)) if us else None}
        out["rows"] = n_batches * a.batch
        ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
