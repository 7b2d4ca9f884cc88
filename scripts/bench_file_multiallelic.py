#!/usr/bin/env python
"""--treat_multiallelics --recalibrate_genotype file to file, on the device file path (ugvc_filter_bgzf_split) and with
--host_io, on a tiled multi-allelic call set:

  one block of tests/multiallelic_data (generated once from a seed, --block-kbp of reference, about 70 records per kbp,
  a third of them multi-allelic or spanned) is tiled with shifted POS over a reference that repeats the block's
  sequence, until there are at least --records records over --contigs contigs.

The model is a gb3 genotype model on the split frame of the test case (tests/util.make_multiallelic_case).  After a
warm-up of both paths, device and --host_io run alternately `--runs` times each.  Prints and writes (to OUT_DIR) one JSON
document: median wall seconds of each path, the device path's eight stage times (ugvc_filter_bgzf_split_stage_ms, summed
over the contigs, from the log), whether the two outputs are byte-identical once inflated, the card's name and power
limit, and the registers / spills ptxas reports for sm_90a for ma_score and the other kernels of csrc/multiallelic.cu
(compiled with -Xptxas -v into a temporary directory).  Needs a CUDA device: there is no CPU fallback.

    python scripts/bench_file_multiallelic.py OUT_DIR [--records N] [--runs K]
"""
import argparse
import json
import logging
import os
import pickle
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def ma_ptxas() -> dict:
    """Registers, stack frame and spills of every kernel of multiallelic.cu as ptxas reports them for sm_90a."""
    csrc = os.path.join(ROOT, "variantcalling_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory(prefix="ptxas_") as tmp:
        r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c",
                            os.path.join(csrc, "multiallelic.cu"), "-o", os.path.join(tmp, "ma.o")], capture_output=True, text=True)
    if r.returncode:
        raise SystemExit("bench_file_multiallelic: nvcc failed on multiallelic.cu:\n" + r.stderr[-2000:])
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for _Z(\d+)(\w+)", line)
        if m:
            name = m.group(2)[: int(m.group(1))]  # the mangled name's length prefix
            cur = name if name.startswith("ma_") else None
            continue
        if cur and "stack frame" in line:
            frame, stores, loads = (int(v) for v in re.findall(r"(\d+) bytes", line)[:3])
            out[cur] = {"stack_bytes": frame, "spill_store_bytes": stores, "spill_load_bytes": loads}
        elif cur and "Used" in line:
            out[cur]["registers"] = int(re.search(r"Used (\d+) registers", line).group(1))
            cur = None
    if "ma_score" not in out:
        raise SystemExit("bench_file_multiallelic: no ptxas report for ma_score")
    return out


def write_input(work: str, n_records: int, n_contigs: int, block_kbp: int, seed: int):
    """-> (vcf path, fasta path, customs, records written)."""
    from tests import multiallelic_data as MD
    from variantcalling_b200 import bgzf_io

    block = block_kbp * 1000
    saved = dict(MD.CONTIGS)
    MD.CONTIGS.clear()
    MD.CONTIGS["blk"] = block
    try:
        t0 = time.perf_counter()
        ds = MD.generate(seed)
        print(f"block: {len(ds['lines'])} records over {block_kbp} kbp in {time.perf_counter() - t0:.1f} s", flush=True)
    finally:
        MD.CONTIGS.clear()
        MD.CONTIGS.update(saved)
    rows = [ln.split("\t", 2) for ln in ds["lines"]]
    tiles = -(-n_records // (len(rows) * n_contigs))
    names = [f"chrT{k + 1}" for k in range(n_contigs)]
    header = [h for h in ds["header"] if not h.startswith("##contig")]
    at = next(i for i, h in enumerate(header) if h.startswith("##INFO") or h.startswith("##FORMAT"))
    header = header[:at] + [f"##contig=<ID={c},length={block * tiles}>" for c in names] + header[at:]
    lines = []
    for c in names:
        for t in range(tiles):
            lines += [f"{c}\t{int(p) + t * block}\t{rest}" for _c, p, rest in rows]
    vcf = os.path.join(work, "in.vcf.gz")
    bgzf_io.write_vcf_gz(vcf, header, lines)
    fasta = os.path.join(work, "ref.fa")
    with open(fasta, "w") as fh:
        fh.write(MD.fasta_text({c: ds["ref"]["blk"] * tiles for c in names}))
    return vcf, fasta, ds["customs"], len(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--contigs", type=int, default=3)
    ap.add_argument("--block-kbp", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seed", type=int, default=8)  # a block the reference splits without raising
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_file_multiallelic: no CUDA device")
    from tests import util
    from variantcalling_b200 import bgzf_io
    from variantcalling_b200 import filter_variants_pipeline as fvp

    os.makedirs(args.out_dir, exist_ok=True)
    ptxas = ma_ptxas()
    print(json.dumps({"multiallelic_ptxas_sm_90a": ptxas}), flush=True)
    work = tempfile.mkdtemp(prefix="filesplit_")
    vcf, fasta, customs, n = write_input(work, args.records, args.contigs, args.block_kbp, args.seed)
    _ds, tr, model, _split = util.make_multiallelic_case(21, "gb3")
    mpath = os.path.join(work, "model.pkl")
    with open(mpath, "wb") as fh:
        pickle.dump({"transformer": tr, "xgb": model}, fh)
    flags = ["--input_file", vcf, "--model_file", mpath, "--treat_multiallelics", "--ref_fasta", fasta, "--recalibrate_genotype"]
    flags += [a for c in customs for a in ("--custom_annotations", c)]
    stage_re = re.compile(r"device split path, ms on the GPU: " + ", ".join([r"[^,]*? (\d+)"] * 8))

    class Grab(logging.Handler):
        def __init__(self):
            super().__init__()
            self.msgs = []

        def emit(self, record):
            self.msgs.append(record.getMessage())

    grab = Grab()
    logging.getLogger(fvp.__name__).addHandler(grab)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    times = {"device": [], "host_io": []}
    stages, fell_back = [], False
    for rep in range(args.runs + 1):  # the first round warms both paths (page cache, allocations, model import)
        for mode in ("device", "host_io"):
            out = os.path.join(work, f"out_{mode}.vcf.gz")
            grab.msgs.clear()
            t0 = time.perf_counter()
            fvp.run(flags + ["--output_file", out] + (["--host_io"] if mode == "host_io" else []))
            dt = time.perf_counter() - t0
            if rep:
                times[mode].append(dt)
            if mode == "device":
                fell_back |= any("taking the host path" in m for m in grab.msgs)
                m = [x for x in (stage_re.search(y) for y in grab.msgs) if x]
                if rep and m:
                    stages.append([int(v) for v in m[-1].groups()])
    same = np.array_equal(bgzf_io.inflate(os.path.join(work, "out_device.vcf.gz")),
                          bgzf_io.inflate(os.path.join(work, "out_host_io.vcf.gz")))
    result = {
        "gpu": smi, "records": n, "contigs": args.contigs, "runs": args.runs,
        "device_s_median": float(np.median(times["device"])), "host_io_s_median": float(np.median(times["host_io"])),
        "device_s": times["device"], "host_io_s": times["host_io"],
        "device_variants_per_s": n / float(np.median(times["device"])),
        "host_io_variants_per_s": n / float(np.median(times["host_io"])),
        "device_stage_ms_median": np.median(np.array(stages), axis=0).tolist() if stages else None,
        "stage_names": ["H2D + inflate", "index K1", "split build", "scored K1..K3", "merge + score", "record writer",
                        "deflate + pack", "D2H"],
        "a_contig_fell_back": fell_back, "same_text": bool(same), "multiallelic_ptxas_sm_90a": ptxas}
    with open(os.path.join(args.out_dir, "bench_file_multiallelic.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))
    shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
