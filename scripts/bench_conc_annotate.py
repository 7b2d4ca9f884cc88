#!/usr/bin/env python
"""annotate_concordance on a synthetic concordance frame: the kernel alone (CUDA events around each launch, over
repeated calls), ConcordanceContext.annotate ("device_call": packing, copies and kernel), the whole annotate_concordance call with its host packing and column
building shown apart, and the oracle's rows/s on a prefix.  Prints one JSON line with the card name and power limit.

  python scripts/bench_conc_annotate.py --rows 5000000 --oracle_rows 100000 --reps 5
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import annotate_ref as AR  # noqa: E402
from tests import annotate_data as AD  # noqa: E402
from variantcalling_b200 import concordance as PC  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=5_000_000)
    ap.add_argument("--oracle_rows", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch

    genome = AD.make_genome(7, {"chr1": 2_000_000, "chr2": 1_000_000, "chr3": 500_000})
    tmp = tempfile.mkdtemp()
    fa = os.path.join(tmp, "g.fa")
    with open(fa, "w") as fh:
        fh.write(AD.fasta_text(genome))
    t0 = time.perf_counter()
    df = AD.make_frame(genome, a.rows, 11)
    t_gen = time.perf_counter() - t0
    ctx = PC.ConcordanceContext(0)
    PC.annotate_concordance(df.head(1000).copy(), fa, ctx=ctx)  # warm-up: contig upload, module load

    # the pieces of one call: host packing, the device call (upload + kernel + download), host columns
    ids = np.array([ctx.annot_contig(fa, c) for c in ("chr1", "chr2", "chr3")], dtype=np.int32)
    codes = df["chrom"].map({"chr1": 0, "chr2": 1, "chr3": 2}).to_numpy()
    refs, alleles = df["ref"].tolist(), df["alleles"].tolist()
    t0 = time.perf_counter()
    ref_b, ref_off = PC._pack_strings(refs)  # noqa: SLF001
    al_b, al_off = PC._pack_strings([x for al in alleles for x in al])  # noqa: SLF001
    t_pack = time.perf_counter() - t0

    dev_ms, kern_ms = [], []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        res = ctx.annotate(ids[codes], df["pos"].to_numpy(), df["indel"].to_numpy(), refs, alleles, "TGCA")
        e.record()
        torch.cuda.synchronize()
        dev_ms.append(s.elapsed_time(e))
        kern_ms.append(float(ctx.lib.ugvc_conc_annot_kernel_ms(ctx.h)))

    t_call = []
    for _ in range(a.reps):
        d = df.copy()
        t0 = time.perf_counter()
        PC.annotate_concordance(d, fa, ctx=ctx)
        t_call.append(time.perf_counter() - t0)

    t0 = time.perf_counter()
    idx = df.index
    PC._object_column(PC._motif_strings(res["left"]), idx)  # noqa: SLF001
    PC._object_column(PC._motif_strings(res["right"]), idx)  # noqa: SLF001
    PC._object_column(PC._INDEL_CLASS[res["class"]], idx)  # noqa: SLF001
    PC._object_column(PC._HMER_NUC[res["hmer_nuc"]], idx)  # noqa: SLF001
    PC._object_column(PC._CYCLE_SKIP[res["cycleskip"]], idx)  # noqa: SLF001
    t_unpack = time.perf_counter() - t0

    sub = df.head(a.oracle_rows)
    t0 = time.perf_counter()
    AR.annotate(sub, genome, "TGCA")
    t_oracle = time.perf_counter() - t0
    out = {
        "card": card(), "rows": a.rows, "frame_build_s": round(t_gen, 2),
        "call_s_median": round(float(np.median(t_call)), 4),
        "kernel_ms_median": round(float(np.median(kern_ms)), 3), "kernel_ms_all": [round(x, 3) for x in kern_ms],
        "device_call_ms_median": round(float(np.median(dev_ms)), 2),
        "host_pack_s": round(t_pack, 4), "host_unpack_s": round(t_unpack, 4),
        "rows_per_s_call": round(a.rows / float(np.median(t_call))),
        "oracle_rows": a.oracle_rows, "oracle_rows_per_s": round(a.oracle_rows / t_oracle),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
