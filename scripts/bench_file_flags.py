#!/usr/bin/env python
"""The CLI file to file in the flag configurations of the reference's system tests (all but --treat_multiallelics), on
the device file path and with --host_io, on one synthetic single-sample .vcf.gz (the configs[1] device generator,
BASELINE.json; 5 M records by default):

  model_bl_cg      model + --blacklist (two blacklists) + --blacklist_cg_insertions
  model_recal      3-class model + --recalibrate_genotype
  bl_only          no model, --blacklist + --blacklist_cg_insertions
  cg_only          no model, --blacklist_cg_insertions

Each configuration runs warm, alternating device / --host_io, `--runs` times each.  Prints and writes (to the directory
given) one JSON document: median variants/s of each, and the device path's stage milliseconds (ugvc_filter_bgzf_stage_ms,
summed over calls, from the log).  Before the runs the record writer's kernels are compiled for sm_90a with
`-Xptxas -v` (into a temporary directory) and their registers, stack and spills go into the JSON too.  Needs a CUDA
device: there is no CPU fallback.

    python scripts/bench_file_flags.py OUT_DIR [--records N] [--runs K]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))


class Blacklist:  # the attribute contract of ugbio_filtering.blacklist.Blacklist
    def __init__(self, blacklist, annotation):
        self.blacklist, self.annotation, self.description = blacklist, annotation, ""
        self.selection_fcn = None


def write_input(work: str, n_records: int, n_custom: int, model, tr, customs):
    """The configs[1] file: device generator -> BGZF + .tbi (as scripts/run_cfg2_cli.py writes it).  Returns the path and
    a sample of (contig, pos) for the blacklists."""
    import torch

    import run_cfg2_cli as cfg2
    from variantcalling_b200 import bgzf_io, lib
    from variantcalling_b200 import model_compiler as MC

    header_text = lib.synth_header(n_custom)
    ctx = lib.Context(0)
    ctx.load_plan(MC.compile_plan(header_text, tr, model, customs).blob)
    idx = lib.Context(0)
    idx.load_plan(MC.compile_plan_no_model(header_text).blob)
    B = 1_000_000
    cap = int(B * 470 * 1.3) + (8 << 20)
    idx.reserve(cap, B + 128, 1)
    d_text = torch.empty(cap, dtype=torch.uint8, device="cuda")
    vcf = os.path.join(work, "in.vcf.gz")
    w = bgzf_io.BgzfWriter(vcf, level=1)
    w.write(header_text.encode())
    names, first = cfg2.contig_of_records(n_records)
    pos_all, end_all, us, ue = [], [], [], []
    for b0 in range(0, n_records, B):
        nb = min(B, n_records - b0)
        nbytes = ctx.synth_device(cfg2.SEED, b0, nb, n_records, n_custom, d_text.data_ptr(), cap - 64)
        torch.cuda.synchronize()
        host = d_text[:nbytes].cpu().numpy()
        res = idx.filter_batch(host)
        base = w.uoffset
        w.write(host)
        ri, ls = res["recinfo"], res["line_start"]
        pos_all.append(ri["pos"].astype(np.int64) - 1)
        end_all.append(ri["pos"].astype(np.int64) - 1 + np.maximum(1, (ri["flags"] >> 8).astype(np.int64)))
        us.append(base + ls[:-1])
        ue.append(base + ls[1:])
    w.close()
    cat = np.concatenate
    contig_idx = (np.searchsorted(first, np.arange(n_records), side="right") - 1).astype(np.int32)
    present = np.unique(contig_idx)
    remap = np.full(len(names), -1, dtype=np.int32)
    remap[present] = np.arange(present.size)
    bgzf_io.write_tbi(vcf + ".tbi", bgzf_io.build_tbi([names[i] for i in present], remap[contig_idx], cat(pos_all), cat(end_all),
                                                     w.virtual_offsets(cat(us)), w.virtual_offsets(cat(ue) - 1) + np.uint64(1)))
    pos = cat(pos_all) + 1
    ctx.close()
    idx.close()
    return vcf, [(names[contig_idx[i]], int(pos[i])) for i in range(0, n_records, 97)]


def writer_ptxas() -> dict:
    """Registers, stack frame and spills of splice_len / splice_copy as ptxas reports them for sm_90a."""
    csrc = os.path.join(ROOT, "variantcalling_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory(prefix="ptxas_") as tmp:
        r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c",
                            os.path.join(csrc, "fileio.cu"), "-o", os.path.join(tmp, "fileio.o")], capture_output=True, text=True)
    if r.returncode:
        raise SystemExit("bench_file_flags: nvcc failed on fileio.cu:\n" + r.stderr[-2000:])
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for _Z\d+(splice_len|splice_copy)", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "stack frame" in line:
            frame, stores, loads = (int(v) for v in re.findall(r"(\d+) bytes", line)[:3])
            out[cur] = {"stack_bytes": frame, "spill_store_bytes": stores, "spill_load_bytes": loads}
        elif cur and "Used" in line:
            out[cur]["registers"] = int(re.search(r"Used (\d+) registers", line).group(1))
            cur = None
    if set(out) != {"splice_len", "splice_copy"}:
        raise SystemExit("bench_file_flags: no ptxas report for the writer kernels")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--records", type=int, default=5_000_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--n-custom", type=int, default=5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_file_flags: no CUDA device")
    import run_cfg2_cli as cfg2
    from sklearn.linear_model import LogisticRegression

    from variantcalling_b200 import bgzf_io
    from variantcalling_b200 import filter_variants_pipeline as fvp

    os.makedirs(args.out_dir, exist_ok=True)
    ptxas = writer_ptxas()
    print(json.dumps({"writer_ptxas_sm_90a": ptxas}), flush=True)
    work = tempfile.mkdtemp(prefix="fileflags_")
    model, tr, customs = cfg2.build_lr_model(args.n_custom)
    vcf, sites = write_input(work, args.records, args.n_custom, model, tr, customs)
    # a 3-class model on the same features (class 2 where the first feature is high)
    from oracle import ref_pipeline as R
    from oracle.vcf_reader import OracleVariantFile
    from variantcalling_b200 import synth

    header, lines, labels = synth.generate(synth.SynthSpec(n_records=20000, n_custom=args.n_custom, seed=1984))
    import pandas as pd

    df = R.get_vcf_df(OracleVariantFile(synth.vcf_text(header, lines)), None, customs)
    with pd.option_context("future.infer_string", False):
        x = tr.transform(R.harness_float_columns(df)).to_numpy(dtype=np.float64)
    y3 = np.where(x[:, 2] > np.median(x[:, 2]), 2, labels)
    model3 = LogisticRegression(max_iter=400).fit(x, y3)
    paths = {}
    for name, obj in (("model", {"transformer": tr, "xgb": model}), ("model3", {"transformer": tr, "xgb": model3}),
                      ("bl", [Blacklist(set(sites[::2]), "ILLUMINA_FP"), Blacklist(set(sites[::3]), "COHORT_FP")])):
        paths[name] = os.path.join(work, name + ".pkl")
        with open(paths[name], "wb") as fh:
            pickle.dump(obj, fh)
    cust = [a for c in customs for a in ("--custom_annotations", c)]
    configs = {
        "model_bl_cg": ["--model_file", paths["model"], "--blacklist", paths["bl"], "--blacklist_cg_insertions"] + cust,
        "model_recal": ["--model_file", paths["model3"], "--recalibrate_genotype"] + cust,
        "bl_only": ["--blacklist", paths["bl"], "--blacklist_cg_insertions"],
        "cg_only": ["--blacklist_cg_insertions"],
    }
    stage_re = re.compile(r"device file path, ms on the GPU: H2D \+ inflate (\d+), K1\.\.K3 (\d+), record writer (\d+), "
                          r"deflate \+ pack (\d+), D2H (\d+)")

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
    result = {"gpu": smi, "records": args.records, "runs": args.runs, "writer_ptxas_sm_90a": ptxas, "configs": {}}
    for name, flags in configs.items():
        times = {"device": [], "host_io": []}
        stages, fell_back = [], False
        for rep in range(args.runs + 1):  # the first round warms both paths (page cache, allocations, model import)
            for mode in ("device", "host_io"):
                out = os.path.join(work, f"out_{name}_{mode}.vcf.gz")
                grab.msgs.clear()
                t0 = time.perf_counter()
                fvp.run(["--input_file", vcf, "--output_file", out] + flags + (["--host_io"] if mode == "host_io" else []))
                dt = time.perf_counter() - t0
                if rep:
                    times[mode].append(dt)
                if mode == "device":
                    fell_back |= any("taking the host path" in m for m in grab.msgs)
                    m = [stage_re.search(x) for x in grab.msgs]
                    m = [x for x in m if x]
                    if rep and m:
                        stages.append([int(v) for v in m[-1].groups()])
        same = np.array_equal(bgzf_io.inflate(os.path.join(work, f"out_{name}_device.vcf.gz")),
                              bgzf_io.inflate(os.path.join(work, f"out_{name}_host_io.vcf.gz")))
        result["configs"][name] = {
            "device_variants_per_s": args.records / float(np.median(times["device"])),
            "host_io_variants_per_s": args.records / float(np.median(times["host_io"])),
            "device_s": times["device"], "host_io_s": times["host_io"],
            "device_stage_ms_median": np.median(np.array(stages), axis=0).tolist() if stages else None,
            "stage_names": ["H2D + inflate", "K1..K3", "record writer", "deflate + pack", "D2H"],
            "a_range_fell_back": fell_back, "same_text": bool(same)}
        print(json.dumps({name: result["configs"][name]}), flush=True)
    with open(os.path.join(args.out_dir, "bench_file_flags.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result))
    shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
