#!/usr/bin/env python
"""Timing of the concordance metrics (BASELINE configs[4]) on one GPU, beside the oracle port of the
reference's pandas / sklearn path on a bounded sample.  Prints one JSON line.

  python scripts/bench_concordance.py [--records 50000000] [--cpu-sample 2000000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=50_000_000)
    ap.add_argument("--cpu-sample", type=int, default=2_000_000)
    ap.add_argument("--repeat", type=int, default=3)
    args = ap.parse_args()
    import torch

    from variantcalling_b200 import concordance as PC
    from variantcalling_b200 import lib

    n = args.records
    rng = np.random.default_rng(1)
    indel = rng.random(n) < 0.25
    hmer = np.where(indel & (rng.random(n) < 0.7), rng.integers(1, 16, size=n), 0).astype(np.int32)
    truth = rng.random(n) < 0.8
    scores = np.clip(rng.normal(np.where(truth, 60, 25), 18), 0, None).astype(np.float32).astype(np.float64)
    cls = np.where(rng.random(n) < 0.03, 2, truth.astype(np.uint8)).astype(np.uint8)
    pred = (scores > 30).astype(np.uint8)  # noqa: PLR2004
    ctx = PC.ConcordanceContext(0)
    out = {"metric": "records/sec through calc_accuracy_metrics + calc_recall_precision_curve", "records": n}

    def timed(fn):
        best = 1e30
        for _ in range(args.repeat):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            best = min(best, time.perf_counter() - t0)
        return best

    t_counts = timed(lambda: ctx.run(scores, pred, cls, indel, hmer, want_curves=False))
    t_all = timed(lambda: ctx.run(scores, pred, cls, indel, hmer, want_curves=True))
    out["host_arrays"] = {"counts_only_s": t_counts, "counts_and_curves_s": t_all, "records_per_s": n / t_all,
                          "h2d_bytes": int(n * (8 + 1 + 1 + 1 + 4))}
    # device-resident inputs
    d = [torch.from_numpy(a).cuda() for a in (scores, pred, cls, indel.astype(np.uint8), hmer)]
    L = lib.load_library()
    counts = np.zeros((PC.N_GROUPS, PC.N_COUNTERS), np.int64)
    clen, cut, sel = np.zeros(9, np.int64), np.zeros(9), np.zeros((9, 2), np.int64)
    p = lib._ptr  # noqa: SLF001

    def device_run(curves):
        rc = L.ugvc_conc_run(ctx.h, n, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), d[4].data_ptr(),
                             None, 1, int(curves), p(counts), p(clen), p(cut), p(sel))
        assert rc == 0, L.ugvc_conc_last_error(ctx.h)

    t_dc = timed(lambda: device_run(False))
    t_da = timed(lambda: device_run(True))
    out["device_arrays"] = {"counts_only_s": t_dc, "counts_and_curves_s": t_da, "records_per_s": n / t_da,
                            "classify_kernel_GBps_incl_alloc": n * 18 / t_dc / 1e9, "curve_points": clen.tolist()}
    # CPU: the oracle port of the reference path on a sample
    import pandas as pd

    from oracle import concordance_ref as CR

    m = min(n, args.cpu_sample)
    df = pd.DataFrame({"filter": np.where(pred[:m] > 0, "PASS", "LOW_SCORE"), "tree_score": scores[:m],
                       "classify": np.array(["fp", "tp", "fn"], dtype=object)[cls[:m]], "indel": indel[:m],
                       "hmer_indel_length": hmer[:m], "hmer_indel_nuc": None})
    t0 = time.perf_counter()
    CR.calc_accuracy_metrics(df, "classify")
    CR.calc_recall_precision_curve(df, "classify")
    t_cpu = time.perf_counter() - t0
    out["cpu_baseline"] = {"kind": "port", "cores": 1, "sample": f"{m} records", "records_per_s": m / t_cpu}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
