#!/usr/bin/env python
"""filter_low_af_ratio_to_background, file to file on the device: warm wall seconds of run(argv) on a generated
tumor/normal VCF (median of alternated runs on the BGZF-with-.tbi and plain-text inputs), records/s, the stage ms of the
device call, and the oracle's records/s on a 100 k prefix.  Usage: python scripts/bench_low_af_ratio.py [--records N]
[--out DIR]; prints one JSON line and writes it to DIR/bench_low_af_ratio.json."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import low_af_ratio_data as D  # noqa: E402
from variantcalling_b200 import bgzf_io, lib  # noqa: E402
from variantcalling_b200 import low_af_ratio as T  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=5_000_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="afr_bench_")
    t0 = time.perf_counter()
    text = D.random_text(a.records, 2, 3, contigs=tuple(f"chr{k}" for k in range(1, 23)))
    gen_s = time.perf_counter() - t0
    head, body = text.split("#CHROM", 1)
    hl = (head + "#CHROM" + body.split("\n", 1)[0]).rstrip("\n").split("\n")
    rl = body.split("\n", 1)[1].rstrip("\n").split("\n")
    src = os.path.join(tmp, "in.vcf.gz")
    bgzf_io.write_vcf_gz(src, hl, rl)
    src_txt = os.path.join(tmp, "in.vcf")
    open(src_txt, "w").write(text)
    argv = lambda s: [s, os.path.join(tmp, "out.vcf.gz"), "--af_ratio_threshold", "10",  # noqa: E731
                      "--af_ratio_threshold_h_indels", "2", "--tumor_vaf_threshold_h_indels", "0.15"]
    T.run(argv(src))  # warm-up: module loads, pinned pools, the device
    times = {"bgzf_tbi": [], "text": []}
    for _ in range(a.runs):
        for key, s in (("bgzf_tbi", src), ("text", src_txt)):
            t = time.perf_counter()
            T.run(argv(s))
            times[key].append(time.perf_counter() - t)
    # stage ms of one device call on the first piece
    ctx = lib.Context(0)
    from variantcalling_b200 import model_compiler as MC
    from variantcalling_b200.vcf_header import VcfHeader

    hdr = VcfHeader("\n".join(hl) + "\n")
    ctx.load_plan(MC.compile_plan_no_model(hdr).blob)
    piece = text.encode()[len("\n".join(hl)) + 1:][: T.PIECE_BYTES]
    piece = piece[: piece.rfind(b"\n") + 1]
    import numpy as np

    buf = np.frombuffer(piece, np.uint8)
    ctx.reserve(buf.size + 64, buf.size // 8 + 16, 1)
    p = T.afr_params(hdr, 10, 2, 0.15, "LowAFRatioToBackground")
    for _ in range(3):
        r = ctx.afr_bgzf(buf, 0, 0, True, p, buf.size // 8 + 16)
    stage = ctx.afr_stage_ms()
    comp = np.frombuffer(bgzf_io.compress_bytes(piece), np.uint8)
    for _ in range(3):
        r = ctx.afr_bgzf(comp, 0, 0, False, p, buf.size // 8 + 16)
    stage_bgzf = ctx.afr_stage_ms()
    ctx.close()
    # the oracle on a 100 k prefix
    from oracle import low_af_ratio_ref as R

    pre = "\n".join(hl) + "\n" + "\n".join(rl[:100_000]) + "\n"
    t = time.perf_counter()
    R.run_text(pre, af_ratio_threshold=10, af_ratio_threshold_h_indels=2, t_vaf_threshold=0.15)
    oracle_rps = 100_000 / (time.perf_counter() - t)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"records": a.records, "input_bytes": len(text), "gpu": gpu, "wall_s": med, "runs": times,
           "records_per_s": {k: a.records / v for k, v in med.items()}, "piece_records": int(r["n_records"]),
           "stage_ms_text_piece": stage, "stage_ms_bgzf_piece": stage_bgzf,
           "stages": ["h2d+inflate", "index K1", "decide+scan+copy", "deflate+pack", "d2h"],
           "oracle_records_per_s": oracle_rps, "generate_s": gen_s}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "bench_low_af_ratio.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
