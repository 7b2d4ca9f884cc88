#!/usr/bin/env python
"""calibrate_bridging_snvs, file to file on the device: warm wall seconds of the whole call on a generated tumor/normal
VCF (BGZF with .tbi) over a seeded multi-contig genome, records/s, the stage ms of the device calls, the FASTA load and
the contig upload timed apart, and the oracle's records/s on a 100 k prefix.  Usage:
python scripts/bench_bridging_snvs.py [--records N] [--out DIR]; prints one JSON line and writes it to
DIR/bench_bridging_snvs.json."""
import argparse
import json
import logging
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import bridging_snvs_data as D  # noqa: E402
from variantcalling_b200 import bgzf_io, lib  # noqa: E402
from variantcalling_b200 import bridging_snvs as T  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=2_000_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    logging.getLogger("variantcalling_b200.bridging_snvs").setLevel(logging.WARNING)  # the log lines are not timed
    tmp = tempfile.mkdtemp(prefix="bsn_bench_")
    contigs = tuple(f"chr{k}" for k in range(1, 9))
    t0 = time.perf_counter()
    g = D.genome(3, tuple((c, 500_000) for c in contigs))
    recs = D.random_records(g, a.records, 4, contigs=contigs)
    gen_s = time.perf_counter() - t0
    head = D.header(contigs=contigs).rstrip("\n").split("\n")
    src = os.path.join(tmp, "in.vcf.gz")
    bgzf_io.write_vcf_gz(src, head, recs)
    ref = os.path.join(tmp, "ref.fa")
    with open(ref, "wb") as fh, open(ref + ".fai", "w") as fai:
        for name, seq in g.items():
            fh.write(b">" + name.encode() + b"\n")
            fai.write(f"{name}\t{len(seq)}\t{fh.tell()}\t60\t61\n")
            for k in range(0, len(seq), 60):
                fh.write(seq[k: k + 60] + b"\n")
    out = os.path.join(tmp, "out.vcf.gz")
    T.calibrate_bridging_snvs(src, ref, out)  # warm-up: module loads, pinned pools, the device
    times = []
    for _ in range(a.runs):
        t = time.perf_counter()
        n_rescued = T.calibrate_bridging_snvs(src, ref, out)
        times.append(time.perf_counter() - t)
    # the FASTA load and the contig upload apart
    t = time.perf_counter()
    fasta = T.load_contigs(ref, src)
    load_s = time.perf_counter() - t
    ctx = lib.Context(0)
    t = time.perf_counter()
    for name, seq in fasta.items():
        ctx.bsn_add_contig(name, seq)
    upload_s = time.perf_counter() - t
    # stage ms of one device call on the first piece
    from variantcalling_b200 import model_compiler as MC
    from variantcalling_b200 import vcf_pieces
    from variantcalling_b200.vcf_header import VcfHeader

    hdr = VcfHeader(bgzf_io.read_header_text(src))
    ctx.load_plan(MC.compile_plan_no_model(hdr).blob)
    inp = vcf_pieces.Input(src, len(bgzf_io.read_header_text(src).encode()), T.PIECE_BYTES)
    data, skip, take, span = inp.pieces[0]
    ctx.reserve(span + 64, span // 8 + 16, 1)
    p = T.bsn_params(hdr)
    stages = []
    for _ in range(5):
        r = ctx.bsn_bgzf(data, skip, take, False, p, span // 8 + 16)
        stages.append(ctx.bsn_stage_ms())
    ctx.close()
    # the oracle on a 100 k prefix
    from oracle import bridging_snvs_ref as R

    pre = "\n".join(head) + "\n" + "\n".join(recs[:100_000]) + "\n"
    t = time.perf_counter()
    R.run_text(pre, g)
    oracle_rps = 100_000 / (time.perf_counter() - t)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    med = statistics.median(times)
    res = {"records": a.records, "rescued": int(n_rescued), "input_bytes": os.path.getsize(src), "gpu": gpu, "wall_s": med,
           "runs": times, "records_per_s": a.records / med, "fasta_load_s": load_s, "contig_upload_s": upload_s,
           "genome_bases": sum(len(v) for v in g.values()), "piece_records": int(r["n_records"]),
           "stage_ms_bgzf_piece": stages[-1], "stages": ["h2d+inflate", "index K1", "decide+scan+copy", "deflate+pack", "d2h"],
           "oracle_records_per_s": oracle_rps, "generate_s": gen_s}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "bench_bridging_snvs.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
