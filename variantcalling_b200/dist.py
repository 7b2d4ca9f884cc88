"""Multi-GPU host logic: contig sharding and the one collective of the path.

Records are independent and the reference already iterates contig by contig
(``filter_variants_pipeline.py:116-120``; its annotator framework shards by contig,
``ugbio_core/vcfbed/variant_annotation.py:159-204``), so ranks own whole contigs
(longest-processing-time bin packing on record counts) and never exchange data;
the only collective is a SUM all-reduce of the int64[4] counter block
{n_records, n_low_score, n_pass, n_cg} -- NCCL over NVLink on GPUs, gloo in the CPU tests.
"""
from __future__ import annotations

import numpy as np


def lpt_partition(loads: dict, world: int) -> list[list]:
    """Assign keys (contigs) with the given loads (record counts) to ``world`` ranks."""
    bins: list[list] = [[] for _ in range(world)]
    total = [0] * world
    for key, load in sorted(loads.items(), key=lambda kv: (-kv[1], str(kv[0]))):
        i = int(np.argmin(total))
        bins[i].append(key)
        total[i] += load
    return bins


def contig_record_ranges(total: int, contig_lengths: dict) -> dict:
    """{contig: (first record, last record)} of a synthetic job of ``total`` records, exactly
    as the device generator lays records out (proportional to contig length)."""
    genome = sum(contig_lengths.values())
    out, cum = {}, 0
    names = list(contig_lengths)
    for i, name in enumerate(names):
        r0 = total * cum // genome
        r1 = total if i == len(names) - 1 else total * (cum + contig_lengths[name]) // genome
        out[name] = (r0, r1)
        cum += contig_lengths[name]
    return out


def allreduce_counts(counts_tensor, group=None):
    """In-place SUM all-reduce of the counter block (a torch tensor on the rank's device)."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(counts_tensor, op=dist.ReduceOp.SUM, group=group)
    return counts_tensor


def bind_to_gpu_numa_node(gpu_index: int) -> dict:
    """Pin this process (and the threads it starts later) to the CPUs of the NUMA node the GPU hangs off, BEFORE any
    pinned host buffer is allocated: first-touch then places those buffers on that node, so the H2D / D2H copies of
    several ranks do not all cross the same memory controller / PCIe root.  Best effort: returns what was done, never raises."""
    import os
    import subprocess

    info = {"gpu": gpu_index, "node": None, "cpus": None}
    try:
        bus = subprocess.run(["nvidia-smi", "--query-gpu=pci.bus_id", "--format=csv,noheader", "-i", str(gpu_index)],
                             capture_output=True, text=True, timeout=20).stdout.strip().lower()
        if not bus:
            return info
        if len(bus.split(":")[0]) == 8:  # 00000000:1B:00.0 -> 0000:1b:00.0
            bus = bus[4:]
        node = int(open(f"/sys/bus/pci/devices/{bus}/numa_node").read().strip())
        if node < 0:
            return info
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        allowed = cpus & os.sched_getaffinity(0)
        if allowed:
            os.sched_setaffinity(0, allowed)
            info.update(node=node, cpus=len(allowed))
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return info
