#!/usr/bin/env python
"""bench.py -- variants/s filtered + scored on the synthetic WGS VCF (BASELINE.json metric).

Workload (config.workload = "cfg3"): BASELINE.json configs[2]/[3] -- N synthetic
single-sample records (default 50 M, SURVEY.md 8d schema, 40 custom annotations =>
81 features), tree-ensemble model 100 trees x depth 6 (sklearn
GradientBoostingClassifier with the reference's XGBClassifier hyper-parameters,
variant_filtering_utils.py:70-78; xgboost is not installed in this image).

  value     records/s with the VCF text already resident in HBM: each timed step is one
            pass of K0..K3 over every record this rank owns (contig-sharded at N > 1,
            one NCCL all-reduce of the pass/fail counters per step).  CUDA events on the
            launching stream, max over ranks.  Inputs (>= 2 GB per rank) exceed L2.
  e2e       the same pass through the host-buffer C-ABI calls (ugvc_submit_batch /
            ugvc_collect_batch): text in pinned host memory, H2D + kernels + D2H of
            flags/probs/qual/recinfo/line_start inside the timed region.
  roofline  for the dominant kernel: algorithmic bytes per launch / mean launch duration
            (CUDA events bracketing each stage inside the timed region) over the measured
            HBM copy peak (MEASURED_PEAKS.json).
  cpu_baseline  the oracle (restated reference CPU path, pandas/sklearn) on a bounded sample.

`--impl reference` times that CPU path alone (rank 0) and prints the same JSON shape.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")

METRIC = "variants/sec filtered+scored on 50M-record synthetic VCF"
SEED = 20260922
N_CUSTOM = 40
FALLBACK_HBM_GBS = 3350.0  # H100 SXM data sheet (HBM3, 3.35 TB/s): used only where no measured peak is present


def log(*a):
    print(*a, file=sys.stderr, flush=True)


_REAL_STDOUT = None


def claim_stdout():
    """stdout must carry exactly one JSON line.  Libraries (NCCL's version banner, for one) write
    to file descriptor 1 directly, so fd 1 is pointed at stderr for the whole run and the JSON line
    is written to the saved descriptor at the end."""
    global _REAL_STDOUT  # noqa: PLW0603
    if _REAL_STDOUT is None:
        sys.stdout.flush()
        _REAL_STDOUT = os.dup(1)
        os.dup2(2, 1)


def emit_json(line: dict):
    data = (json.dumps(line) + "\n").encode()
    sys.stdout.flush()
    if _REAL_STDOUT is None:
        os.write(1, data)
    else:
        os.write(_REAL_STDOUT, data)


# ------------------------------------------------------------------------------------------
def build_model(n_train: int = 20000):
    """Train the cfg-3 model on host-generated records of the same schema."""
    import pandas as pd

    from oracle import ref_pipeline as R  # training frame only (CPU, like train_models_pipeline)
    from oracle.vcf_reader import OracleVariantFile
    from sklearn.ensemble import GradientBoostingClassifier
    from variantcalling_b200 import synth
    from variantcalling_b200 import transformers as T
    from variantcalling_b200.tprep_constants import VcfType

    spec = synth.SynthSpec(n_records=n_train, n_custom=N_CUSTOM, seed=1984)
    header, lines, labels = synth.generate(spec)
    customs = synth.custom_annotation_names(N_CUSTOM)
    vf = OracleVariantFile(synth.vcf_text(header, lines))
    df = R.get_vcf_df(vf, None, customs)
    tr = T.get_transformer(VcfType.SINGLE_SAMPLE, [c.lower() for c in customs])
    with pd.option_context("future.infer_string", False):
        x = tr.fit_transform(R.harness_float_columns(df)).to_numpy(dtype=np.float64)
    np.random.seed(1984)
    model = GradientBoostingClassifier(n_estimators=100, learning_rate=0.15, subsample=0.4, max_depth=6,
                                       random_state=0)
    model.fit(x, labels)
    return model, tr, customs


def contig_record_ranges(total: int):
    """[ (contig index, first record, last record) ] exactly as the device generator lays them out."""
    from variantcalling_b200.synth import CONTIG_LENGTHS

    lens = list(CONTIG_LENGTHS.values())
    genome = sum(lens)
    out, cum = [], 0
    for c, ln in enumerate(lens):
        r0 = total * cum // genome
        r1 = total if c == len(lens) - 1 else total * (cum + ln) // genome
        out.append((c, r0, r1))
        cum += ln
    return out


def range_partition(ranges, world: int):
    """Equal record ranges in genome order: rank r owns records [r N / W, (r + 1) N / W), cut into (contig, first, last)
    pieces at the contig borders (a piece never spans contigs: a batch is lines of one contig, as in the tool).  Whole
    contigs by LPT left rank 0 three per cent above the mean at eight ranks; ranges are exact."""
    total = ranges[-1][2]
    bins = []
    for r in range(world):
        lo, hi = total * r // world, total * (r + 1) // world
        bins.append([(c, max(r0, lo), min(r1, hi)) for c, r0, r1 in ranges if min(r1, hi) > max(r0, lo)])
    return bins


def lpt_partition(ranges, world: int):
    """Longest-processing-time bin packing of contigs onto ranks (SURVEY.md 8e)."""
    bins = [[] for _ in range(world)]
    load = [0] * world
    for c, r0, r1 in sorted(ranges, key=lambda t: t[2] - t[1], reverse=True):
        i = int(np.argmin(load))
        bins[i].append((c, r0, r1))
        load[i] += r1 - r0
    return [sorted(b) for b in bins]


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.gpu = gpu_index
        self.rows = []
        self.proc = None
        self.thread = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.gpu)], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.proc = None
            return
        self.thread = threading.Thread(target=self._read, daemon=True)
        self.thread.start()

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self) -> dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx = float(r[2])
            except (ValueError, IndexError):
                continue
            names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
            for name, val in zip(names, r[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        # under load = samples at or above the median of the upper half
        load = sorted(sm)[len(sm) // 2:] if sm else []
        return {"sm_mhz": float(np.median(load)) if load else None, "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm)}


# ------------------------------------------------------------------------------------------
def run_reference(args):
    """The reference's CPU implementation of the path (oracle port), rank 0 only."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import multiprocessing as mp

    from variantcalling_b200 import synth

    cores = min(os.cpu_count() or 1, 64)
    per_worker = args.cpu_sample_per_worker
    n_sample = cores * per_worker
    log(f"[reference] building model + {n_sample} sample records on the host")
    model, tr, customs = build_model()
    spec = synth.SynthSpec(n_records=n_sample, n_custom=N_CUSTOM, seed=SEED)
    header, lines, _ = synth.generate(spec)
    chunks = [(header, lines[i * per_worker:(i + 1) * per_worker], model, tr, customs) for i in range(cores)]
    ctx = mp.get_context("fork")
    times = []
    with ctx.Pool(cores) as pool:
        for it in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            done = pool.map(_reference_worker, chunks)
            dt = time.perf_counter() - t0
            assert sum(done) == n_sample
            if it >= args.warmup:
                times.append(dt)
            log(f"[reference] iter {it}: {n_sample / dt:.0f} variants/s")
    total = sum(times)
    value = n_sample * len(times) / total
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": "variants/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * total / len(times),
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": {"workload": "cfg3: synthetic WGS VCF, 81 features, 100x depth-6 tree ensemble",
                   "sample_records_per_step": n_sample},
        "cpu_baseline": {"value": value, "unit": "variants/s", "cores": cores, "kind": "port",
                         "sample": f"{n_sample} records per step ({per_worker} per worker process), the reference's "
                                   f"pandas/sklearn path restated in oracle/ (pysam/xgboost absent)",
                         "note": "the parse / write stages are a pure-Python stand-in for htslib's C code (about half of "
                                 "this arm's time): a baseline beside the GPU number, not the real reference's speed"},
        "e2e": {"value": value, "unit": "variants/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    emit_json(line)


def _reference_worker(job):
    header, lines, model, tr, customs = job
    from oracle import ref_pipeline as R
    from oracle.vcf_reader import OracleVariantFile
    from variantcalling_b200 import synth

    vf = OracleVariantFile(synth.vcf_text(header, lines))
    res = R.filter_variants(vf, model, tr, custom_annotations=customs)
    return len(res["lines"])


def _parity_worker(job):
    header_text, text, model, tr, customs = job
    from oracle import ref_pipeline as R
    from oracle.vcf_reader import OracleVariantFile

    vf = OracleVariantFile((header_text + text.decode()).encode())
    res = R.filter_variants(vf, model, tr, custom_annotations=customs)
    low = np.array(["LOW_SCORE" in f.split(";") for f in res["filters"]])
    return low, np.asarray(res["probs"], dtype=np.float64)


def spread_parity(chunks, header_text, model, tr, customs, workers):
    """FILTER / probabilities of the oracle on record chunks taken all along the input (worker processes: the
    pandas path does about 10^4 records a second per core)."""
    import multiprocessing as mp

    jobs = [(header_text, c, model, tr, customs) for c in chunks]
    with mp.get_context("fork").Pool(workers) as pool:  # the children only run NumPy / pandas / sklearn
        return pool.map(_parity_worker, jobs)


def cpu_baseline_sample(text: bytes, header_text: str, model, tr, customs) -> dict:
    """Oracle timed single-process (like the reference's serial contig loop) on a bounded sample."""
    from oracle import ref_pipeline as R
    from oracle.vcf_reader import OracleVariantFile

    vf = OracleVariantFile((header_text + text.decode()).encode())
    tm = {}
    t0 = time.perf_counter()
    res = R.filter_variants(vf, model, tr, custom_annotations=customs, timings=tm)
    dt = time.perf_counter() - t0
    n = len(res["lines"])
    return {"value": n / dt, "unit": "variants/s", "cores": 1, "kind": "port",
            "sample": f"first {n} records of the bench input, single process; stage seconds: "
                      + ", ".join(f"{k}={v:.2f}" for k, v in tm.items()),
            "note": "pysam / htslib and xgboost are absent from the image: the parse and write stages run a pure-Python "
                    "stand-in for htslib's C reader / writer (oracle/vcf_reader.py), the model is sklearn's -- the real "
                    "reference spends less time in those stages", "_res": res}


DUMP_SEED = 7
DUMP_MAX_RECORDS = 1 << 20
DUMP_MAX_BYTES = 64 << 20


def dump_outputs(out_dir: str, d_low, d_probs, d_qual, counts):
    """What the caller of the device-resident path receives (FILTER flag, class probabilities, TREE_SCORE and the
    pass/fail counters), for the same seeded sample of records in every run.  float32 / float64 only."""
    import torch

    n, k = d_probs.shape
    per_record = 8 + 4 + 4 * k + 8  # index, low_score, probs, qual
    m = min(n, DUMP_MAX_RECORDS, (DUMP_MAX_BYTES - 4096) // per_record)
    idx = np.sort(np.random.default_rng(DUMP_SEED).choice(n, size=m, replace=False))
    idx_t = torch.from_numpy(idx).to(d_low.device)
    arrays = {
        "record_index": idx.astype(np.float64),
        "low_score": d_low.index_select(0, idx_t).cpu().numpy().astype(np.float32),
        "probs": d_probs.index_select(0, idx_t).cpu().numpy().astype(np.float32),
        "qual": d_qual.index_select(0, idx_t).cpu().numpy().astype(np.float64),
        "counts": np.asarray(counts, dtype=np.float64),
    }
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, f"{name}.npy"), a)
    log(f"[bench] outputs of the last step: {m} of {n} records -> {out_dir} "
        f"({sum(a.nbytes for a in arrays.values()) / 2**20:.1f} MiB)")


# ------------------------------------------------------------------------------------------
def main():  # noqa: C901, PLR0912, PLR0915
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--records", type=int, default=50_000_000, help="total records of the job (all ranks)")
    ap.add_argument("--batch-records", type=int, default=2_000_000)
    ap.add_argument("--cpu-sample", type=int, default=120_000, help="records timed on the CPU oracle at N=1 (about 15 s)")
    ap.add_argument("--cpu-sample-per-worker", type=int, default=8000)
    ap.add_argument("--parity-records", type=int, default=1_024_000,
                    help="records checked against the oracle, in 64 chunks spread over the whole input (N=1, needs the e2e pass)")
    ap.add_argument("--e2e-steps", type=int, default=0, help="timed e2e steps (0 = same as --steps)")
    ap.add_argument("--lanes", type=int, default=3)
    ap.add_argument("--min-presence", type=float, default=None, help="learn_key_order presence threshold (profiling)")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--e2e-bgzf", action="store_true",
                    help="also time the e2e pass with BGZF-compressed host buffers inflated on the device "
                         "(ugvc_submit_bgzf; adds an e2e_bgzf object; on by default at N=1)")
    ap.add_argument("--no-e2e-bgzf", action="store_true")
    ap.add_argument("--no-e2e-file", action="store_true",
                    help="skip the file-to-file leg (BASELINE configs[1] through `ugvc filter_variants_pipeline`, N=1 only)")
    ap.add_argument("--e2e-file-records", type=int, default=5_000_000)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last device-resident step returned (rank 0's records) "
                         "as DIR/<name>.npy: a fixed, seeded sample of at most 1 Mi records")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if int(os.environ.get("WORLD_SIZE", "1")) == 1 and not args.no_e2e and not args.no_e2e_bgzf:
        args.e2e_bgzf = True
    claim_stdout()
    if args.warmup < 3:  # noqa: PLR2004
        args.warmup = 3
    if args.impl == "reference":
        run_reference(args)
        return

    import torch

    from variantcalling_b200 import lib
    from variantcalling_b200 import model_compiler as MC

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (there is no CPU fallback for the hot path)")
    from variantcalling_b200 import dist as vdist

    numa = vdist.bind_to_gpu_numa_node(local_rank) if world > 1 else {"gpu": local_rank, "node": None, "cpus": None}
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist  # noqa: PLC0415

        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))

    # ---- model + plan (identical on every rank: seeded)
    t0 = time.perf_counter()
    model, tr, customs = build_model()
    header_text = lib.synth_header(N_CUSTOM)
    plan = MC.compile_plan(header_text, tr, model, customs)
    if rank == 0:
        log(f"[bench] model+plan in {time.perf_counter() - t0:.1f}s: F={plan.n_features} slots={plan.n_slots} "
            f"plan={len(plan.blob)} B")
    ctx = lib.Context(local_rank)
    ctx.load_plan(plan.blob)
    K = ctx.n_classes

    # ---- this rank's records: contigs by LPT, generated straight into HBM in batches
    ranges = contig_record_ranges(args.records)
    mine = range_partition(ranges, world)[rank]
    n_mine = sum(r1 - r0 for _, r0, r1 in mine)
    B = min(args.batch_records, max(1, n_mine))
    bytes_guess = int(n_mine * 470 * 1.05) + (64 << 20)
    d_text = torch.empty(bytes_guess, dtype=torch.uint8, device="cuda")
    ctx.reserve(int(B * 470 * 1.3) + (8 << 20), B, args.lanes)
    batches = []  # (byte offset, n_bytes, n_records)
    off = 0
    # a non-default torch stream: its handle is non-zero, so the C ABI launches on exactly the
    # stream the torch CUDA events below are recorded on
    work_stream = torch.cuda.Stream()
    torch.cuda.set_stream(work_stream)
    stream = work_stream.cuda_stream
    assert stream != 0
    for _, r0, r1 in mine:
        for b0 in range(r0, r1, B):
            nb = min(B, r1 - b0)
            nbytes = ctx.synth_device(SEED, b0, nb, args.records, N_CUSTOM, d_text.data_ptr() + off,
                                      bytes_guess - off - 64, stream)
            batches.append((off, nbytes, nb))
            off += (nbytes + 255) // 256 * 256  # keep every batch 256-byte aligned
    total_bytes = sum(b[1] for b in batches)
    torch.cuda.synchronize()
    if rank == 0:
        log(f"[bench] rank0: {n_mine} records, {total_bytes / 1e9:.2f} GB text in HBM, {len(batches)} batches, "
            f"mean line {total_bytes / max(1, n_mine):.1f} B")
    # the usual INFO key order / FORMAT column, learned from the head of the input like the CLI does
    head = bytes(d_text[batches[0][0]: batches[0][0] + min(batches[0][1], 1 << 20)].cpu().numpy())
    kw = {} if args.min_presence is None else {"min_presence": args.min_presence}
    info_order, fmt_order = lib.learn_key_order(head[: head.rfind(b"\n") + 1], **kw)
    ctx.set_key_order(info_order, fmt_order)
    max_b = max(b[2] for b in batches)
    d_low = torch.empty(n_mine, dtype=torch.uint8, device="cuda")
    d_probs = torch.empty((n_mine, K), dtype=torch.float32, device="cuda")
    d_qual = torch.empty(n_mine, dtype=torch.float64, device="cuda")
    d_nrec = torch.zeros(len(batches), dtype=torch.int64, device="cuda")

    class _Raw:  # CUDA array interface over the context's int64[4] counter block
        def __init__(self, ptr):
            self.__cuda_array_interface__ = {"shape": (4,), "typestr": "<i8", "data": (ptr, False), "version": 2}

    counts_t = torch.as_tensor(_Raw(ctx.counts_device_ptr()), device="cuda")

    def device_pass():
        rec0 = 0
        for bi, (boff, nbytes, nb) in enumerate(batches):
            ctx.filter_device(d_text.data_ptr() + boff, nbytes, 30.0, d_low.data_ptr() + rec0,
                              d_probs.data_ptr() + rec0 * K * 4, d_qual.data_ptr() + rec0 * 8, nb,
                              d_n_records=d_nrec.data_ptr() + bi * 8, stream=stream)
            rec0 += nb
        if dist is not None:  # the single collective of the path: pass/fail counters
            dist.all_reduce(counts_t, op=dist.ReduceOp.SUM)

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- device-resident measurement
    for _ in range(args.warmup):
        counts_t.zero_()
        device_pass()
    barrier()
    ctx.device_status(stream)  # surfaces data errors loudly
    assert int(d_nrec.sum().item()) == n_mine, "record count mismatch between generator and line index"
    launches0 = ctx.launch_count()
    ctx.enable_stage_timing(True)
    sampler = ClockSampler(local_rank)
    sampler.start()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    ev0.record()
    for _ in range(args.steps):
        counts_t.zero_()
        device_pass()
    ev1.record()
    barrier()
    clocks = sampler.stop()
    elapsed_ms = ev0.elapsed_time(ev1)
    stage_sum, n_calls = ctx.stage_ms()
    ctx.enable_stage_timing(False)
    slow_last = ctx.slow_records(0)  # records of the last batch that went through the generic parser (-1: tile kernel off)
    launches = ctx.launch_count() - launches0
    counts_total = [int(v) for v in counts_t.tolist()]
    t_el = torch.tensor([elapsed_ms], dtype=torch.float64, device="cuda")
    if dist is not None:
        dist.all_reduce(t_el, op=dist.ReduceOp.MAX)
    elapsed_ms = float(t_el.item())
    value = args.records * args.steps / (elapsed_ms / 1e3)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, d_low, d_probs, d_qual, counts_total)

    # ---- roofline of the dominant kernel (this rank's launches)
    peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(peaks_path):
        peak, peak_src = float(json.load(open(peaks_path))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    else:
        peak, peak_src = FALLBACK_HBM_GBS, "fallback: H100 SXM data-sheet HBM3 bandwidth, not a measured peak"
    names = ["k0_line_index", "k1_field_parse", "k2_feature_assembly", "k3_inference"]
    S, F = ctx.n_slots, ctx.n_features
    rec_per_launch = n_mine / len(batches)
    text_per_launch = total_bytes / len(batches)
    alg_bytes = {  # algorithmic (compulsory) bytes per launch, DESIGN.md section 3
        "k0_line_index": text_per_launch + 8 * rec_per_launch,
        "k1_field_parse": text_per_launch + rec_per_launch * (8 + 4 * S + 16),
        "k2_feature_assembly": rec_per_launch * 4 * (S + F),
        "k3_inference": rec_per_launch * (4 * F + 4 * K + 9),  # fused K2+K3: one 4-byte slot read per feature
    }
    stage_ms = {n: stage_sum[i] / max(1, n_calls) for i, n in enumerate(names)}
    dom = max(names, key=lambda n: stage_ms[n])
    achieved = alg_bytes[dom] / (stage_ms[dom] / 1e3) / 1e9
    path_bytes = total_bytes / max(1, n_mine) + 4 * K + 9  # B_alg per record, SURVEY.md 8d
    kernels_ms_per_step = sum(stage_sum) / args.steps
    # DRAM bytes per record of each kernel, where a summary of `ncu --set full` captures taken on this GPU model is
    # present (profiles/ncu_traffic.json: {kernel: {"dram_bytes": dram__bytes_read.sum + dram__bytes_write.sum of one
    # launch, "records": the records that launch parsed}}); None otherwise
    traffic_path = os.path.join(ROOT, "profiles", "ncu_traffic.json")
    ncu_traffic = json.load(open(traffic_path)) if os.path.exists(traffic_path) else {}
    stage_kernel = {"k1_field_parse": "k1_tok", "k3_inference": "k3_heap", "k2_feature_assembly": "k2_features",
                    "k0_line_index": "k0_index"}

    def traffic_of(stage):
        t = ncu_traffic.get(stage_kernel.get(stage, ""))
        return None if not t else t["dram_bytes"] / t["records"] * rec_per_launch

    per_kernel = {}
    for nme in names:
        if stage_ms[nme] > 1e-3:  # stages folded into another kernel report no time
            ach = alg_bytes[nme] / (stage_ms[nme] / 1e3) / 1e9
            per_kernel[nme] = {"ms_per_launch": stage_ms[nme], "algorithmic_bytes_per_launch": alg_bytes[nme],
                               "achieved": ach, "frac": ach / peak, "traffic": traffic_of(nme)}
    roofline = {"bound": "hbm", "kernel": dom, "achieved": achieved, "peak": peak, "unit": "GB/s",
                "frac": achieved / peak, "traffic": traffic_of(dom),
                "traffic_source": "profiles/ncu_traffic.json (ncu --set full, dram bytes of one launch / its records, "
                                  "scaled to this launch size)" if traffic_of(dom) is not None else None,
                "algorithmic_bytes_per_launch": alg_bytes[dom], "peak_source": peak_src,
                "stage_ms_per_launch": stage_ms, "launches_timed": n_calls, "per_kernel": per_kernel,
                "stages": "k0 (line index) is folded into k1's tile kernel, k2 (feature assembly) into k3's tile load: "
                          "their own stages read ~0 ms",
                "path": {"bytes_per_record": path_bytes,
                         "achieved": path_bytes * n_mine / (kernels_ms_per_step / 1e3) / 1e9,
                         "frac": path_bytes * n_mine / (kernels_ms_per_step / 1e3) / 1e9 / peak}}

    # ---- e2e through the host-buffer C ABI
    e2e = None
    if not args.no_e2e:
        h_text = lib.PinnedBuffer(off + 64)
        t_view = torch.from_numpy(h_text.array)
        t_view[:off].copy_(d_text[:off])
        torch.cuda.synchronize()
        RI = lib.RECINFO_DTYPE.itemsize
        h_out = lib.PinnedBuffer(n_mine * (1 + 4 * K + 8 + RI) + (n_mine + len(batches)) * 8 + 64)
        arr = h_out.array
        p = 0
        o_low = arr[p:p + n_mine]; p += n_mine  # noqa: E702
        p = (p + 7) // 8 * 8
        o_probs = arr[p:p + n_mine * 4 * K].view(np.float32).reshape(n_mine, K); p += n_mine * 4 * K  # noqa: E702
        o_qual = arr[p:p + n_mine * 8].view(np.float64); p += n_mine * 8  # noqa: E702
        o_ri = arr[p:p + n_mine * RI].view(lib.RECINFO_DTYPE); p += n_mine * RI  # noqa: E702
        o_ls = arr[p:p + (n_mine + len(batches)) * 8].view(np.int64)
        text_ptr = h_text.ptr
        n_lanes = args.lanes

        def host_pass():
            rec_of = []
            rec0 = 0
            for boff, nbytes, nb in batches:
                rec_of.append(rec0)
                rec0 += nb
            inflight = []
            got = 0
            for bi, (boff, nbytes, nb) in enumerate(batches):
                lane = bi % n_lanes
                if len(inflight) == n_lanes:
                    got += _collect(inflight.pop(0))
                ctx.submit(lane, text_ptr + boff, nbytes, 30.0)
                inflight.append((lane, bi))
            while inflight:
                got += _collect(inflight.pop(0))
            return got

        rec_starts = np.cumsum([0] + [b[2] for b in batches])

        def _collect(item):
            lane, bi = item
            r0, nb = int(rec_starts[bi]), batches[bi][2]
            out = {"low_score": o_low[r0:r0 + nb], "probs": o_probs[r0:r0 + nb], "qual": o_qual[r0:r0 + nb],
                   "recinfo": o_ri[r0:r0 + nb], "line_start": o_ls[r0 + bi:r0 + bi + nb + 1]}
            return ctx.collect(lane, out, nb)

        e_steps = args.e2e_steps or args.steps
        for _ in range(2):
            assert host_pass() == n_mine
        barrier()
        t0 = time.perf_counter()
        for _ in range(e_steps):
            host_pass()
        barrier()
        dt = time.perf_counter() - t0
        t_e = torch.tensor([dt], dtype=torch.float64, device="cuda")
        if dist is not None:
            dist.all_reduce(t_e, op=dist.ReduceOp.MAX)
        dt = float(t_e.item())
        d2h = n_mine * (1 + 4 * K + 8 + RI) + (n_mine + len(batches)) * 8
        e2e = {"value": args.records * e_steps / dt, "unit": "variants/s", "h2d_bytes_per_step": int(total_bytes),
               "d2h_bytes_per_step": int(d2h), "steps": e_steps, "lanes": n_lanes,
               "api": "ugvc_submit_batch/ugvc_collect_batch (pinned host buffers)"}
        # consistency: host path == device path
        assert np.array_equal(o_low, d_low.cpu().numpy()), "host-buffer path differs from the device-resident path"

    # ---- parity along the whole input (N=1): 64 record chunks, one per stretch of the batch list, oracle in worker processes
    parity = None
    if e2e is not None and rank == 0 and world == 1 and not args.no_cpu_baseline and args.parity_records > 0:
        n_chunks = 64
        per = max(1, args.parity_records // n_chunks)
        picks, chunks = [], []
        for c in range(n_chunks):
            bi = c * len(batches) // n_chunks
            boff, _nbytes, nb = batches[bi]
            r0b = int(rec_starts[bi])
            n_c = min(per, nb)
            first = (c * 7919) % max(1, nb - n_c + 1)  # a different place inside every batch
            ls = o_ls[r0b + bi: r0b + bi + nb + 1]
            b0, b1 = int(ls[first]), int(ls[first + n_c])
            chunks.append(bytes(h_text.array[boff + b0: boff + b1]))
            picks.append((r0b + first, n_c))
        t0 = time.perf_counter()
        res = spread_parity(chunks, header_text, model, tr, customs, min(os.cpu_count() or 1, 64))
        same, worst, n_checked = True, 0.0, 0
        for (g0, n_c), (low, pr) in zip(picks, res):
            same &= bool(np.array_equal(low, o_low[g0:g0 + n_c].astype(bool)))
            worst = max(worst, float(np.abs(pr - o_probs[g0:g0 + n_c]).max()))
            n_checked += n_c
        parity = {"records": n_checked, "chunks": n_chunks, "filter_identical": same, "max_abs_prob_diff": worst,
                  "seconds": time.perf_counter() - t0,
                  "what": "oracle (reference CPU path restated) vs the e2e results, chunks spread over all batches"}
        log(f"[bench] parity on {n_checked} records in {n_chunks} chunks: FILTER identical={same}, max |dp|={worst:.2e}")
        assert same, "FILTER differs from the oracle on the spread sample"

    # ---- e2e with compressed host buffers (opt-in): the host ships BGZF blocks, the device inflates them
    e2e_bgzf = None
    if args.e2e_bgzf and not args.no_e2e:
        from variantcalling_b200 import bgzf_io

        t0 = time.perf_counter()
        parts = [bgzf_io.compress_bytes(h_text.array[boff:boff + nbytes], level=6) for boff, nbytes, _nb in batches]
        len_of = [len(c) for c in parts]  # exact compressed size of each batch (the buffer pads batches to 64 bytes)
        comp_off = np.concatenate(([0], np.cumsum([(len(c) + 63) // 64 * 64 for c in parts]))).astype(np.int64)
        h_comp = lib.PinnedBuffer(int(comp_off[-1]) + 64)
        for c, o in zip(parts, comp_off[:-1]):
            h_comp.array[o:o + len(c)] = np.frombuffer(c, dtype=np.uint8)
        comp_bytes = int(sum(len(c) for c in parts))
        if rank == 0:
            log(f"[bench] e2e_bgzf: {total_bytes / 1e9:.2f} GB of text -> {comp_bytes / 1e9:.2f} GB of BGZF "
                f"in {time.perf_counter() - t0:.1f}s on the host (not timed)")
        del parts

        def bgzf_pass():
            inflight, got = [], 0
            for bi in range(len(batches)):
                lane = bi % n_lanes
                if len(inflight) == n_lanes:
                    got += _collect(inflight.pop(0))
                ctx.submit_bgzf(lane, h_comp.ptr + int(comp_off[bi]), len_of[bi], 30.0)
                inflight.append((lane, bi))
            while inflight:
                got += _collect(inflight.pop(0))
            return got

        o_low[:] = 0
        for _ in range(2):
            assert bgzf_pass() == n_mine
        assert np.array_equal(o_low, d_low.cpu().numpy()), "compressed-input path differs from the device-resident path"
        barrier()
        t0 = time.perf_counter()
        for _ in range(e_steps):
            bgzf_pass()
        barrier()
        dt = time.perf_counter() - t0
        t_e = torch.tensor([dt], dtype=torch.float64, device="cuda")
        if dist is not None:
            dist.all_reduce(t_e, op=dist.ReduceOp.MAX)
        e2e_bgzf = {"value": args.records * e_steps / float(t_e.item()), "unit": "variants/s",
                    "h2d_bytes_per_step": comp_bytes, "d2h_bytes_per_step": int(d2h), "steps": e_steps, "lanes": n_lanes,
                    "compression_ratio": total_bytes / comp_bytes,
                    "api": "ugvc_submit_bgzf/ugvc_collect_batch (BGZF level 6 in pinned host buffers, inflated on the device)"}

    # ---- CPU baseline on a bounded sample of the same input (rank 0, N=1)
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        n_s = min(args.cpu_sample, batches[0][2])
        ls = torch.empty(batches[0][2] + 1, dtype=torch.int64, device="cuda")
        tmp_low = torch.empty(batches[0][2], dtype=torch.uint8, device="cuda")
        tmp_p = torch.empty((batches[0][2], K), dtype=torch.float32, device="cuda")
        tmp_q = torch.empty(batches[0][2], dtype=torch.float64, device="cuda")
        ctx.filter_device(d_text.data_ptr() + batches[0][0], batches[0][1], 30.0, tmp_low.data_ptr(),
                          tmp_p.data_ptr(), tmp_q.data_ptr(), batches[0][2], stream=stream,
                          d_line_start=ls.data_ptr())
        torch.cuda.synchronize()
        end = int(ls[n_s].item())
        sample_text = bytes(d_text[batches[0][0]: batches[0][0] + end].cpu().numpy())
        cpu = cpu_baseline_sample(sample_text, header_text, model, tr, customs)
        res = cpu.pop("_res")
        want_low = np.array(["LOW_SCORE" in f.split(";") for f in res["filters"]])
        got_low = tmp_low[:n_s].cpu().numpy().astype(bool)
        cpu["filter_parity_on_sample"] = bool(np.array_equal(want_low, got_low))
        cpu["max_abs_prob_diff_on_sample"] = float(np.abs(res["probs"] - tmp_p[:n_s].cpu().numpy()).max())

    # ---- file to file through the drop-in CLI (BASELINE.md section 4's clock: .vcf.gz in -> .vcf.gz + .tbi out), N=1:
    # BASELINE configs[1] (5 M records, logistic regression) in a child process that writes the input, runs
    # filter_variants_pipeline.run twice in-process and once as a fresh `python ugvc ...`, and checks the output
    e2e_file = None
    if rank == 0 and world == 1 and not args.no_e2e and not args.no_e2e_file:
        import subprocess
        import tempfile
        del d_text
        torch.cuda.empty_cache()
        with tempfile.TemporaryDirectory(prefix="bench_cfg2_") as work:
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "run_cfg2_cli.py"), "--records",
                                str(args.e2e_file_records), "--runs", "2", "--workdir", work], capture_output=True, text=True,
                               check=False)
            try:
                d = json.loads(r.stdout.strip().splitlines()[-1])
                ck = d.get("checks", {})
                e2e_file = {"value": d["variants_per_s_file_to_file"], "unit": "variants/s", "records": d["records"],
                            "workload": d["config"], "wall_s": d["cli_wall_s"], "wall_s_runs": d["cli_wall_s_runs"],
                            "fresh_process_wall_s": d.get("cli_process_wall_s"),
                            "fresh_process_variants_per_s": d.get("variants_per_s_process"),
                            "input_file_bytes": d["input_file_bytes"], "output_file_bytes": d["output_file_bytes"],
                            "checks_ok": bool(ck) and "error" not in ck and all(v for k, v in ck.items() if isinstance(v, bool)),
                            "checks": ck, "timing_note": d.get("timing_note"), "leg_seconds": time.perf_counter() - t0}
            except Exception as e:  # noqa: BLE001
                e2e_file = {"error": f"{type(e).__name__}: {e}", "stderr_tail": r.stderr[-600:]}

    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": "variants/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": elapsed_ms / args.steps, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "f64 accumulate / f32 features", "data": "synthetic",
            "config": {"workload": "cfg3: synthetic WGS VCF, 81 features, 100x depth-6 tree ensemble "
                                   "(sklearn GradientBoosting, reference XGB hyper-parameters)",
                       "records_total": args.records, "records_rank0": n_mine, "batch_records": B,
                       "mean_line_bytes": total_bytes / max(1, n_mine),
                       "sharding": "equal record ranges in genome order, pieces cut at contig borders",
                       "l2": "inputs larger than L2 (no flush needed)", "threshold": 30.0,
                       "k1_slow_records_last_batch": slow_last, "numa_binding": numa},
            "clocks": clocks, "e2e": e2e, "gpu_launches": int(launches), "roofline": roofline, "cpu_baseline": cpu,
            "parity": parity,
            **({"e2e_bgzf": e2e_bgzf} if e2e_bgzf is not None else {}),
            **({"e2e_file": e2e_file} if e2e_file is not None else {}),
            "counts_last_steps": {"n_records": counts_total[0], "n_low_score": counts_total[1],
                                  "n_pass": counts_total[2], "n_cg": counts_total[3]},
        }
        emit_json(line)
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
