#!/usr/bin/env python
"""Where K3's time goes on the bench workload: K3 time per launch against the number of trees, and in every k3_heap
shape, on one batch of the bench's records.

    python scripts/k3_budget.py --out DIR [--launches 24] [--shapes] [--tree-shape N]

The bench model (bench.build_model) is compiled truncated to its first n trees (estimators_[:n]) for n in TREES.
Each point runs in a child process (UGVC_K3_SHAPE is read once per process): the first bench batch (generated on
the device from the bench seed) goes through filter_device warm-up launches, then `--launches` timed ones with
stage timing on; K3's figure is the CUDA events around its own launch, summed over the timed launches and divided
by their number.  The tree points run the shape k3_choose picks for each (it can differ between them) or, with
--tree-shape, the one K3H_SHAPES entry given; a line ms = a + b * trees is fitted by least squares over the points that
ran the full model's shape: a is the per-tile cost (tile fetch, K2, k3_finish, barriers, tail), b the walk and leaf
sums of one tree.  --shapes also times the full model in every K3H_SHAPES entry (K3_BUDGET_SHAPES: a list of them).
Writes DIR/k3_budget.json with the card name, power limit and SM clocks read in the same run."""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
TREES = [1, 25, 50, 100]  # sklearn's boosting model cannot be cut to zero stages
SHAPES = [int(v) for v in os.environ.get("K3_BUDGET_SHAPES", "0,1,2,3,4,5,6,7,8,9").split(",")]

_CHILD = r"""
import json, sys
import torch
sys.path.insert(0, sys.argv[1])
import bench
from variantcalling_b200 import lib
blob, n_rec, launches = open(sys.argv[2], "rb").read(), int(sys.argv[3]), int(sys.argv[4])
ctx = lib.Context(0)
try:
    ctx.load_plan(blob)
except lib.UgvcError as e:
    print(json.dumps({"error": e.message}))
    sys.exit(0)
cap = int(n_rec * 470 * 1.3) + (8 << 20)
ctx.reserve(cap, n_rec, 1)
d_text = torch.empty(cap, dtype=torch.uint8, device="cuda")
s = torch.cuda.Stream()
torch.cuda.set_stream(s)
nbytes = ctx.synth_device(bench.SEED, 0, n_rec, 50_000_000, bench.N_CUSTOM, d_text.data_ptr(), cap - 64, s.cuda_stream)
torch.cuda.synchronize()
head = bytes(d_text[: min(nbytes, 1 << 20)].cpu().numpy())
ctx.set_key_order(*lib.learn_key_order(head[: head.rfind(b"\n") + 1]))
K = ctx.n_classes
d_low = torch.empty(n_rec, dtype=torch.uint8, device="cuda")
d_probs = torch.empty((n_rec, K), dtype=torch.float32, device="cuda")
d_qual = torch.empty(n_rec, dtype=torch.float64, device="cuda")
run = lambda: ctx.filter_device(d_text.data_ptr(), nbytes, 30.0, d_low.data_ptr(), d_probs.data_ptr(), d_qual.data_ptr(),
                                n_rec, stream=s.cuda_stream)
for _ in range(5):
    run()
torch.cuda.synchronize()
ctx.device_status(s.cuda_stream)
ctx.enable_stage_timing(True)
for _ in range(launches):
    run()
st, n = ctx.stage_ms()
ctx.enable_stage_timing(False)
print(json.dumps({"cfg": ctx.k3_config(), "k3_ms": st[3] / n, "k1_ms": st[1] / n, "launches": n,
                  "qual_sum": float(d_qual.sum().item())}))
ctx.close()
"""


def _truncated(model, n):
    m = copy.deepcopy(model)
    m.estimators_ = model.estimators_[:n].copy()
    m.n_estimators_ = n
    m.n_estimators = max(n, 1)
    return m


def _child(blob_path, n_rec, launches, env_extra):
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, blob_path, str(n_rec), str(launches)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    if r.returncode != 0:
        return {"error": r.stderr[-2000:]}
    return json.loads(r.stdout.strip().splitlines()[-1])


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (v.strip() for v in out.split(","))))
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--launches", type=int, default=24)
    ap.add_argument("--shapes", action="store_true", help="also time the full model in every K3H_SHAPES entry")
    ap.add_argument("--tree-shape", type=int, default=None, help="K3H_SHAPES entry of the tree points (default: k3_choose's)")
    args = ap.parse_args()
    if args.launches < 20:
        ap.error("--launches: at least 20")
    import bench
    from variantcalling_b200 import lib
    from variantcalling_b200 import model_compiler as MC

    os.makedirs(args.out, exist_ok=True)
    model, tr, customs = bench.build_model()
    header_text = lib.synth_header(bench.N_CUSTOM)
    # the bench's first batch: the first contig's first --batch-records (2 M) records, or the contig if shorter
    _, r0, r1 = bench.contig_record_ranges(50_000_000)[0]
    n_rec = min(2_000_000, r1 - r0)
    res = {"gpu": _gpu_info(), "records_per_launch": n_rec, "launches": args.launches, "trees": {}, "shapes": {}}
    with tempfile.TemporaryDirectory() as tmp:
        blobs = {}
        for n in TREES:
            p = os.path.join(tmp, f"plan{n}.bin")
            with open(p, "wb") as fh:
                fh.write(MC.compile_plan(header_text, tr, _truncated(model, n), customs).blob)
            blobs[n] = p
        for n in TREES:
            env = {} if args.tree_shape is None else {"UGVC_K3_SHAPE": str(args.tree_shape)}
            res["trees"][str(n)] = _child(blobs[n], n_rec, args.launches, env)
            print(n, "trees:", res["trees"][str(n)], flush=True)
        if args.shapes:
            for i in SHAPES:  # entry 8 is entry 1 walking twelve trees at once
                env = {"UGVC_K3_SHAPE": "1", "UGVC_K3_NCH448": "12"} if i == 8 else {"UGVC_K3_SHAPE": str(i)}
                res["shapes"][str(i)] = _child(blobs[TREES[-1]], n_rec, args.launches, env)
                print("shape", i, res["shapes"][str(i)], flush=True)
    full_cfg = res["trees"][str(TREES[-1])].get("cfg", {})
    same = ("kernel", "tpb", "groups", "split")
    pts = [(n, v["k3_ms"]) for n, v in ((int(k), v) for k, v in res["trees"].items())
           if "k3_ms" in v and all(v["cfg"].get(k) == full_cfg.get(k) for k in same)]
    if len(pts) >= 2:
        x, y = np.array([p[0] for p in pts], float), np.array([p[1] for p in pts], float)
        b, a = np.polyfit(x, y, 1)
        full = res["trees"][str(TREES[-1])]["k3_ms"]
        res["fit"] = {"points": pts, "intercept_ms": a, "slope_ms_per_tree": b,
                      "intercept_share_at_full_model": a / full, "slope_share_at_full_model": b * TREES[-1] / full}
    res["gpu_after"] = _gpu_info()
    with open(os.path.join(args.out, "k3_budget.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res.get("fit", {})))


if __name__ == "__main__":
    main()
