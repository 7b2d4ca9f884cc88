#!/usr/bin/env python
"""gvcf_hcr on the device: warm wall seconds of gvcf_hcr (merged BED) and gvcf_to_bed on a generated DeepVariant-like
gVCF (BGZF with .tbi), records/s, the stage ms of the device calls of one piece, the longest reset-to-reset segment
over all pieces, and the oracle's records/s on a 100 k prefix.  The input is generated with NumPy (reference blocks of
geometric length, SNVs, insertions, deletions whose following records overlap them, RefCall deletions) so that 20 M
records fit in one run.  Usage: python scripts/bench_gvcf_hcr.py [--records N] [--out DIR]; prints one JSON line and
writes it to DIR/bench_gvcf_hcr.json."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import gvcf_hcr_data as D  # noqa: E402
from variantcalling_b200 import bgzf_io  # noqa: E402
from variantcalling_b200 import gvcf_hcr as T  # noqa: E402

CONTIGS = ("chr1", "chr2", "chr3", "chr4", "chr5", "chr6", "chr7", "chr8")


def generate(n: int, seed: int) -> tuple[list[str], np.ndarray, np.ndarray, np.ndarray]:
    """(lines, contig index, POS - 1, index end) of n records over CONTIGS."""
    rng = np.random.default_rng(seed)
    kind = np.searchsorted(np.cumsum([0.70, 0.12, 0.05, 0.07, 0.06]), rng.random(n), side="right")
    ln = np.where(rng.random(n) < 0.8, rng.geometric(0.02, n), rng.integers(1, 4, n))
    dl = rng.integers(2, 41, n)
    gq = np.where(rng.random(n) < 0.6, rng.integers(0, 100, n), rng.integers(15, 26, n))
    adv = np.select([kind == 0, kind == 3], [np.where(rng.random(n) < 0.97, ln, np.maximum(1, ln - 2)),
                                             np.where(rng.random(n) < 0.7, 1, dl)], 1)
    cid = np.minimum((np.arange(n) * len(CONTIGS)) // n, len(CONTIGS) - 1)
    first = np.r_[True, cid[1:] != cid[:-1]]
    csum = np.cumsum(adv) - adv
    run0 = np.maximum.accumulate(np.where(first, np.arange(n), 0))
    pos = csum - csum[run0] + 1
    refs = ["A" * int(k) for k in range(42)]
    names = list(CONTIGS)
    lines = []
    for c, p, k, L, d, g in zip(cid.tolist(), pos.tolist(), kind.tolist(), ln.tolist(), dl.tolist(), gq.tolist()):
        if k == 0:
            lines.append(f"{names[c]}\t{p}\t.\tA\t<*>\t0\t.\tEND={p + L - 1}\tGT:GQ:MIN_DP:PL\t0/0:{g}:20:0,{g},99")
        elif k == 1:
            lines.append(f"{names[c]}\t{p}\t.\tA\tC,<*>\t20.5\tPASS\t.\tGT:GQ:DP:PL\t0/1:{g}:25:30,0,40")
        elif k == 2:
            lines.append(f"{names[c]}\t{p}\t.\tA\tATT,<*>\t20.5\tPASS\t.\tGT:GQ:DP:PL\t1/1:{g}:25:30,0,40")
        elif k == 3:
            lines.append(f"{names[c]}\t{p}\t.\t{refs[d]}\tA,<*>\t20.5\tPASS\t.\tGT:GQ:DP:PL\t0/1:{g}:25:30,0,40")
        else:
            lines.append(f"{names[c]}\t{p}\t.\t{refs[d]}\tA,<*>\t0\tRefCall\t.\tGT:GQ:DP:PL\t./.:{g}:25:30,0,40")
    beg = pos - 1
    end = beg + np.select([kind == 0, kind >= 3], [ln, dl], 1)
    return lines, cid, beg, end


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=20_000_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="hcr_bench_")
    t0 = time.perf_counter()
    lines, cid, beg, end = generate(a.records, 5)
    head = D.header(contigs=tuple((c, 300_000_000) for c in CONTIGS))
    src = os.path.join(tmp, "in.g.vcf.gz")
    w = bgzf_io.BgzfWriter(src)
    hdr = ("\n".join(head) + "\n").encode()
    w.write(hdr)
    body = ("\n".join(lines) + "\n").encode()
    w.write(body)
    w.close()
    lens = np.fromiter((len(x) + 1 for x in lines), np.int64, len(lines))
    u0 = len(hdr) + np.cumsum(lens) - lens
    bgzf_io.write_tbi(src + ".tbi", bgzf_io.build_tbi(list(CONTIGS), cid, beg, end, w.virtual_offsets(u0),
                                                      w.virtual_offsets(u0 + lens - 1) + np.uint64(1)))
    gen_s = time.perf_counter() - t0
    del body
    out = os.path.join(tmp, "out.bed")
    T.gvcf_hcr(src, out)  # warm-up: module loads, the device
    times, times_bed = [], []
    for _ in range(a.runs):  # the two calls alternated
        t = time.perf_counter()
        T.gvcf_hcr(src, out)
        times.append(time.perf_counter() - t)
        t = time.perf_counter()
        skipped = T.gvcf_to_bed(src, out + ".1")
        times_bed.append(time.perf_counter() - t)
    n_lines = sum(1 for _ in open(out))
    # every piece through the two device calls on one lane: stage ms and the longest segment
    from variantcalling_b200 import lib, vcf_pieces
    from variantcalling_b200 import model_compiler as MC
    from variantcalling_b200.vcf_header import VcfHeader

    header_text = bgzf_io.read_header_text(src)
    vh = VcfHeader(header_text)
    inp = vcf_pieces.Input(src, len(header_text.encode()), T.PIECE_BYTES, index_cuts=False)
    cap = max(p[3] for p in inp.pieces) + 64
    ctx = lib.Context(0)
    ctx.load_plan(MC.compile_plan_no_model(vh).blob)
    ctx.reserve(cap, cap // 8 + 16, 1)
    p = T.hcr_params(vh, 20, True, True)
    longest, stages, piece_records, last, extent = 0, [], 0, None, -1
    for data, skip, take, span in inp.pieces:
        sc = ctx.hcr_scan(data, skip, take, p, cap // 8 + 16)
        u = inp.starts[len(stages)] + int(sc["runs"][0][1])
        first = inp.text(u, u + 64).split(b"\t", 1)[0].decode()
        em = ctx.hcr_emit(p, first == last, extent, span + 48 * sc["n_records"] + 64)
        last = inp.text(inp.starts[len(stages)] + int(sc["runs"][-1][1]), inp.starts[len(stages)] + int(sc["runs"][-1][1]) + 64)
        last = last.split(b"\t", 1)[0].decode()
        extent = em["exit_extent"]
        longest = max(longest, em["longest_segment"])
        stages.append(ctx.hcr_stage_ms())
        piece_records = max(piece_records, sc["n_records"])
    ctx.close()
    # the oracle on a 100 k prefix
    from oracle import gvcf_hcr_ref as R

    pre = "\n".join(head) + "\n" + "\n".join(lines[:100_000]) + "\n"
    t = time.perf_counter()
    R.run_text(pre, 20, True, do_merge=True)
    oracle_rps = 100_000 / (time.perf_counter() - t)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    med, med_bed = statistics.median(times), statistics.median(times_bed)
    res = {"records": a.records, "input_bytes": os.path.getsize(src), "gpu": gpu, "gvcf_hcr_wall_s": med, "runs": times,
           "records_per_s": a.records / med, "gvcf_to_bed_wall_s": med_bed, "gvcf_to_bed_runs": times_bed,
           "skipped": int(skipped), "merged_lines": n_lines, "pieces": len(inp.pieces), "piece_records": piece_records,
           "longest_segment": longest, "stage_ms_first_piece": stages[0], "stage_ms_median": np.median(stages, 0).tolist(),
           "stages": ["h2d+inflate", "index K1", "decide+prefix max", "emit", "d2h"],
           "oracle_records_per_s": oracle_rps, "generate_s": gen_s}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "bench_gvcf_hcr.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
