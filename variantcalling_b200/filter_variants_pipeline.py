#!/env/python
"""POST-GATK variant filtering -- H100-native drop-in for the reference tool.

Mirrors ``ugbio_utils/src/filtering/ugbio_filtering/filter_variants_pipeline.py``:
same flags (``parse_args``, :20-70), same ``run(argv)`` entry (argv without the
program name, :78-80), same model-pickle contract (``mf["xgb"]``,
``mf["transformer"]``, :89-94), same header edits (:106-113), same contig
iteration (header order or ``--limit_to_contigs``; empty contigs skipped,
:116-127), same FILTER / TREE_SCORE / QUAL / BLACKLST rules (:188-228), same
log lines incl. ``Variant filtering run: success|failed`` and re-raise (:233-240).

What differs is where the work happens: per contig the bgzip'ed text is inflated
by the multi-threaded C++ reader, shipped to the GPU in batches through
``ugvc_submit_batch`` / ``ugvc_collect_batch`` (K0 line index, K1 field parse,
K2 feature assembly, K3 inference + score + decision), and the output lines are
spliced from the original bytes and BGZF-compressed on the host; the ``.tbi`` is
written directly (the reference shells out to ``bcftools index -t``, :231).

``--recalibrate_genotype``: K3 keeps the per-class phreds and the splicer rewrites GT / GQ / PL of
the first sample (:203-215).  ``--treat_multiallelics`` (:145-166): per contig, an index pass
(K0+K1) finds the multi-allelic records and deletion clusters, their biallelic split rows are
written as VCF lines (``variantcalling_b200/multiallelics.py``) and scored by the same kernels with
the untouched records; the fp64 likelihoods are merged per record.  On the device file path all of
that runs in one call per contig (``ugvc_filter_bgzf_split``); ``--host_io`` merges and scores on the host.
"""
from __future__ import annotations

import argparse
import ctypes as C
import logging
import os.path
import pickle
import queue
import sys
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from variantcalling_b200 import bgzf_io, lib, multiallelics
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader


def parse_args(argv: list[str]) -> argparse.Namespace:
    ap_var = argparse.ArgumentParser(prog="filter_variants_pipeline.py", description="Filter VCF")
    ap_var.add_argument("--input_file", help="Name of the input VCF file (requires .tbi index)", type=str,
                        required=True)
    ap_var.add_argument("--model_file", help="Pickle model file", type=str, required=False)
    ap_var.add_argument("--blacklist", help="Blacklist file", type=str, required=False)
    ap_var.add_argument("--custom_annotations",
                        help="Custom INFO annotations to read from the VCF (multiple possible)", required=False,
                        type=str, default=None, action="append")
    ap_var.add_argument("--blacklist_cg_insertions", help="Should CCG/GGC insertions be filtered out?",
                        action="store_true")
    ap_var.add_argument("--treat_multiallelics",
                        help="Should special treatment be applied to multiallelic and spanning deletions",
                        default=False, action="store_true")
    ap_var.add_argument("--recalibrate_genotype", help="Use if the model allows to re-call genotype", default=False,
                        action="store_true")
    ap_var.add_argument("--overwrite_qual_tag", help="Write the score to QUAL field in addition to TREE_SCORE/GQ",
                        default=False, action="store_true")
    ap_var.add_argument("--decision_threshold", help="Decision threshold for filtering variants (default: 30)",
                        type=float, default=30.0)
    ap_var.add_argument("--ref_fasta", help="Reference FASTA file (only required for multiallelic treatment)",
                        required=False, type=str)
    ap_var.add_argument("--output_file", help="Output VCF file", type=str, required=True)
    ap_var.add_argument("--limit_to_contigs", help="Limit filtering to these contigs", nargs="+", type=str,
                        default=None)
    # host knobs (not in the reference; defaults need no tuning)
    ap_var.add_argument("--device", help="CUDA device index (default: LOCAL_RANK or 0)", type=int, default=None)
    ap_var.add_argument("--host_io", help="Inflate, edit and deflate the records on host threads even when the device-side "
                        "file path applies", action="store_true")
    ap_var.add_argument("--batch_mb", help="VCF text per GPU batch, MiB", type=int, default=256)
    ap_var.add_argument("--io_threads", help="Host threads for BGZF inflate/deflate/splice (0 = all)", type=int,
                        default=0)
    return ap_var.parse_args(argv)


def _load_pickle(path: str):
    with open(path, "rb") as fh:
        return pickle.load(fh)  # noqa: S301  (the reference's own contract, :91)


def _blacklist_positions(blacklists, contig: str) -> list[tuple[str, np.ndarray]]:
    """[(annotation, sorted positions on this contig)] from reference-style Blacklist objects
    (``blacklist.py:10-55``: ``.blacklist`` is a set of (chrom, pos), ``.annotation`` a name)."""
    out = []
    for bl in blacklists:
        sel = getattr(bl, "selection_fcn", None)
        name = getattr(sel, "__name__", "") or getattr(sel, "name", "") or str(sel)
        if sel is not None and "ALL" not in str(name).upper() and not getattr(bl, "select_all", False):
            raise NotImplementedError(
                f"blacklist {bl.annotation!r}: only selection_fcn = VariantSelectionFunctions.ALL is lowered")
        pos = np.fromiter((p for (c, p) in bl.blacklist if c == contig), dtype=np.int64)
        out.append((bl.annotation, np.sort(pos)))
    return out



def info_end_positions(text: np.ndarray, line_start: np.ndarray, recinfo: np.ndarray, n: int, n_threads: int = 0) -> np.ndarray:
    """INFO/END of every record (0 where there is none): htslib's tabix for VCF ends a record at END when the tag
    is present and lies beyond POS -- gVCF blocks, symbolic <DEL> / <CNV> alleles -- so that region queries that
    overlap only the tail of a long record find it (`bcftools index -t`, filter_variants_pipeline.py:231).
    One threaded pass over the INFO columns in C (csrc/hostio.cpp: ugvc_info_end)."""
    out = np.zeros(n, dtype=np.int64)
    if n == 0:
        return out
    text = np.ascontiguousarray(text, dtype=np.uint8)
    line_start = np.ascontiguousarray(line_start, dtype=np.int64)
    recinfo = np.ascontiguousarray(recinfo)
    rc = lib.load_library().ugvc_info_end(text.ctypes.data, line_start.ctypes.data, recinfo.ctypes.data, n, out.ctypes.data,
                                          n_threads)
    if rc < 0:
        raise OSError(f"ugvc_info_end failed (ugvc code {rc})")
    return out


class _Splicer:
    """Output side: splice + BGZF append + bookkeeping for the tabix index."""

    def __init__(self, path: str, threads: int):
        self.writer = bgzf_io.BgzfWriter(path, n_threads=threads)
        self.threads = threads
        self.names: list[str] = []
        self.contig_of, self.beg, self.end, self.u_start, self.u_end = [], [], [], [], []
        # tabix sections are built contig by contig on the writer thread (single-process runs), beside the GPU passes
        self.sections: list[bytes] = []
        self._cur: list[tuple] = []
        self.index_info_end = False  # the header declares INFO/END: records end there in the index (htslib's rule)
        self.keep_arrays = False  # multi-rank runs: rank 0 shifts the virtual offsets, so the arrays travel instead
        self.L = lib.load_library()
        self.seconds = {"splice": 0.0, "deflate": 0.0}
        self.ranges: dict[str, tuple[int, int]] = {}  # contig -> [first, last) compressed byte of its blocks
        # BGZF compression + index bookkeeping run on their own thread, in submission order, so that
        # the next batch's GPU pass and splice overlap the previous batch's deflate (zlib releases the GIL)
        self._queue: "queue.Queue" = queue.Queue(maxsize=3)
        self._error: BaseException | None = None
        self._thread = threading.Thread(target=self._drain, name="ugvc-bgzf-writer", daemon=True)
        self._thread.start()
        self._index_pool = ThreadPoolExecutor(max_workers=1, thread_name_prefix="ugvc-tabix")  # sections, in contig order

    def _drain(self):
        while True:
            item = self._queue.get()
            try:
                if item is None:
                    return
                if self._error is None:
                    self._write_spliced(*item)
            except BaseException as err:  # noqa: BLE001  (re-raised on the caller's thread)
                self._error = err
            finally:
                self._queue.task_done()

    def _check_writer(self):
        if self._error is not None:
            err, self._error = self._error, None
            raise err

    def write_header(self, lines: list[str]):
        self.writer.write(("\n".join(lines) + "\n").encode())

    def write_batch(self, contig: str, text: np.ndarray, res: dict, *, with_model: bool, overwrite_qual: bool,
                    bl_code, bl_table: bytes, bl_off: np.ndarray, phreds: np.ndarray | None = None):
        n = res["n_records"]
        if n == 0:
            return
        max_bl = int(np.diff(bl_off).max()) if bl_off is not None and bl_off.size > 1 else 0
        cap = int(text.size + n * (96 + max_bl + (16 * phreds.shape[1] if phreds is not None else 0)) + 1024)
        out = np.empty(cap, dtype=np.uint8)
        out_ls = np.empty(n + 1, dtype=np.int64)
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
        table = np.frombuffer(bl_table, dtype=np.uint8) if bl_code is not None and bl_table else None
        t_splice = time.perf_counter()
        nb = self.L.ugvc_splice_records(
            p(text), p(res["line_start"]), p(res["recinfo"]), p(res.get("low_score")), p(res.get("qual")), n,
            int(overwrite_qual), int(with_model), p(bl_code), p(table), p(bl_off) if table is not None else None,
            p(phreds), 0 if phreds is None else int(phreds.shape[1]), p(out), out.size, p(out_ls), self.threads)
        if nb < 0:
            raise OSError(f"splice failed (ugvc code {nb})")
        self.seconds["splice"] += time.perf_counter() - t_splice
        ri = res["recinfo"]
        beg = ri["pos"].astype(np.int64) - 1
        self._check_writer()
        end = beg + np.maximum(1, (ri["flags"] >> 8).astype(np.int64))
        if self.index_info_end:
            info_end = info_end_positions(text, res["line_start"], ri, n, self.threads)
            end = np.where(info_end > beg, info_end, end)  # htslib ignores an END that is not beyond POS
        self._queue.put((contig, out[:nb], n, beg, end, out_ls))

    def write_device_batch(self, contigs: list[str], bounds: np.ndarray, res: dict, release=None):
        """Records edited and BGZF-compressed on the device (lib.Context.filter_bgzf): only file and index work is left.
        The batch holds the records of `contigs` in order, contig k in [bounds[k], bounds[k + 1]).  `release` is called
        once the buffers of `res` are no longer needed."""
        n = res["n_records"]
        if n == 0:
            if release:
                release()
            return
        ri = res["recinfo"]
        beg = ri["pos"].astype(np.int64) - 1
        self._check_writer()
        end = beg + np.maximum(1, (ri["flags"] >> 8).astype(np.int64))
        if self.index_info_end:
            end = np.where(res["end"] > beg, res["end"], end)  # the INFO/END the device writer read; the rule of write_batch
        self._queue.put(((list(contigs), np.asarray(bounds, dtype=np.int64)), (res["bgzf"], res["block_csize"], release), n, beg,
                         end, res["line_start"]))

    def _write_spliced(self, contig, data, n: int, beg: np.ndarray, end: np.ndarray, out_ls: np.ndarray):
        t0 = time.perf_counter()
        base = self.writer.uoffset
        c_before = self.writer.coffset
        if isinstance(data, tuple):  # compressed on the device
            self.writer.write_compressed(data[0], data[1], int(out_ls[-1]), lib.DEF_CHUNK)
        else:
            self.writer.write(data)
        contigs, bounds = contig if isinstance(contig, tuple) else ([contig], np.array([0, n], dtype=np.int64))
        if len(contigs) == 1:  # (multi-rank runs: always; rank 0 copies the contig's blocks as they are)
            self.ranges[contigs[0]] = (self.ranges.get(contigs[0], (c_before, 0))[0], self.writer.coffset)
        if not self.keep_arrays:
            vs = self.writer.virtual_offsets(base + out_ls[:-1])
            ve = self.writer.virtual_offsets(base + out_ls[1:] - 1) + np.uint64(1)
        for k, name in enumerate(contigs):
            r0, r1 = int(bounds[k]), int(bounds[k + 1])
            if r1 <= r0:
                continue
            if not self.names or self.names[-1] != name:
                self._close_section()
                self.names.append(name)
            if self.keep_arrays:
                self.contig_of.append(np.full(r1 - r0, len(self.names) - 1, dtype=np.int32))
                self.beg.append(beg[r0:r1])
                self.end.append(end[r0:r1])
                self.u_start.append(base + out_ls[r0:r1])
                self.u_end.append(base + out_ls[r0 + 1:r1 + 1])
            else:
                self._cur.append((beg[r0:r1], end[r0:r1], vs[r0:r1], ve[r0:r1]))
        self.seconds["deflate"] += time.perf_counter() - t0
        if isinstance(data, tuple) and data[2] is not None:
            data[2]()  # the device batch's buffers may be reused

    def _close_section(self):
        if self.keep_arrays or not self.names:
            return
        cur, self._cur = self._cur, []

        def section():
            t0 = time.perf_counter()
            cat = np.concatenate
            cols = [cat([c[k] for c in cur]) if cur else np.zeros(0, np.int64) for k in range(4)]
            sec = bgzf_io.tbi_section(cols[0], cols[1], cols[2].astype(np.uint64), cols[3].astype(np.uint64))
            self.seconds["index"] = self.seconds.get("index", 0.0) + time.perf_counter() - t0
            return sec

        self.sections.append(self._index_pool.submit(section))

    def _finish_writer(self):
        self._queue.put(None)
        self._thread.join()
        self._check_writer()

    def abort(self):
        """Stop the writer thread after a failure on the caller's side (the partial file stays)."""
        if self._thread.is_alive():
            self._error = self._error or RuntimeError("aborted")
            self._queue.put(None)
            self._thread.join(timeout=30)

    def finish_part(self) -> dict:
        """Multi-rank runs: this rank's records are on disk (no header, no EOF block, no index); return
        what rank 0 needs to place each contig's blocks in the final file and index them."""
        self._finish_writer()
        meta = {"names": list(self.names), "ranges": dict(self.ranges), "n_bytes": self.writer.coffset}
        if self.contig_of:
            cat = np.concatenate
            us, ue = cat(self.u_start), cat(self.u_end)
            meta.update(contig_of=cat(self.contig_of), beg=cat(self.beg), end=cat(self.end),
                        vs=self.writer.virtual_offsets(us), ve=self.writer.virtual_offsets(ue - 1) + np.uint64(1))
        return meta

    def close(self, path: str):
        self._finish_writer()
        self.writer.close()
        self._close_section()
        bgzf_io.write_tbi(path + ".tbi", bgzf_io.tbi_assemble(self.names, [f.result() for f in self.sections]))
        self._index_pool.shutdown()


class _PinnedPool:
    """A few reusable sets of pinned host buffers (page-locked once, not page-faulted per contig): the compressed
    input of a contig, and what comes back from ugvc_filter_bgzf.  acquire() blocks until a set is free."""

    def __init__(self, n_sets: int):
        self._free: "queue.Queue" = queue.Queue()
        for _ in range(n_sets):
            self._free.put({})

    def acquire(self, sizes: dict, grow: float = 1.0) -> dict:
        """`grow`: how much larger than this request the largest one is expected to be (buffers are sized for that when
        they have to be page-locked, so that they are page-locked once)."""
        bufs = self._free.get()
        for key, (n_items, dtype) in sizes.items():
            need = int(n_items) * np.dtype(dtype).itemsize
            have = bufs.get(key)
            if have is None or have[0].array.size < need:
                if have is not None:
                    have[0].free()
                pb = lib.PinnedBuffer(int(need * max(1.0, grow)) + need // 16 + 4096)
                bufs[key] = (pb, None)
            pb = bufs[key][0]
            bufs[key] = (pb, pb.array[: need].view(dtype))
        return bufs

    def release(self, bufs: dict):
        self._free.put(bufs)


def _part_path(output_file: str, rank: int) -> str:
    return f"{output_file}.rank{rank}.part"


def _assemble_parts(output_file: str, header_lines: list[str], contigs: list[str], world: int, threads: int):
    """Rank 0 of a multi-rank run: header + every contig's BGZF blocks (copied verbatim from the rank
    that owns the contig, in output contig order) + EOF block, and one .tbi over the shifted virtual
    offsets.  BGZF blocks are self-contained, so concatenating whole blocks is a valid BGZF file
    (the reference's own precedent: ``bcftools concat --naive``, variant_annotation.py:96-110)."""
    metas = []
    for r in range(world):
        with open(_part_path(output_file, r) + ".meta", "rb") as fh:
            metas.append(pickle.load(fh))  # noqa: S301  (written by this program a moment ago)
    w = bgzf_io.BgzfWriter(output_file, n_threads=threads)
    w.write(("\n".join(header_lines) + "\n").encode())
    pos = w.coffset
    names, contig_of, beg, end, vs, ve = [], [], [], [], [], []
    with open(output_file, "ab") as dst:
        for contig in contigs:
            owner = next((r for r, m in enumerate(metas) if contig in m["ranges"]), None)
            if owner is None or contig in names:
                continue
            m = metas[owner]
            c0, c1 = m["ranges"][contig]
            with open(_part_path(output_file, owner), "rb") as src:
                src.seek(c0)
                left = c1 - c0
                while left > 0:
                    chunk = src.read(min(left, 64 << 20))
                    if not chunk:
                        raise OSError(f"{_part_path(output_file, owner)} is shorter than its index says")
                    dst.write(chunk)
                    left -= len(chunk)
            sel = np.flatnonzero(m["contig_of"] == m["names"].index(contig))
            shift = pos - c0

            def moved(v, shift=shift):
                block = (v >> np.uint64(16)).astype(np.int64) + shift
                return (block.astype(np.uint64) << np.uint64(16)) | (v & np.uint64(0xFFFF))

            contig_of.append(np.full(sel.size, len(names), dtype=np.int32))
            names.append(contig)
            beg.append(m["beg"][sel])
            end.append(m["end"][sel])
            vs.append(moved(m["vs"][sel]))
            ve.append(moved(m["ve"][sel]))
            pos += c1 - c0
        dst.write(bgzf_io.BGZF_EOF)
    cat = np.concatenate
    if names:
        payload = bgzf_io.build_tbi(names, cat(contig_of), cat(beg), cat(end), cat(vs), cat(ve))
    else:
        z = np.zeros(0, np.int64)
        payload = bgzf_io.build_tbi([], z, z, z, z.astype(np.uint64), z.astype(np.uint64))
    bgzf_io.write_tbi(output_file + ".tbi", payload)
    for r in range(world):
        for suffix in ("", ".meta"):
            try:
                os.remove(_part_path(output_file, r) + suffix)
            except OSError:
                pass


def _split_batches(text: np.ndarray, limit: int):
    """Yield [begin, end) byte ranges of whole lines, each at most ``limit`` bytes (a single
    longer line becomes its own batch)."""
    n, b = text.size, 0
    while b < n:
        e = min(n, b + limit)
        if e < n:
            # the last newline of the window, looked for in growing tails (a line is a few hundred bytes: the first
            # 64 KiB tail nearly always holds one -- no scan of the whole window)
            cut, span = -1, 1 << 16
            while cut < 0:
                lo = max(b, e - span)
                nl = np.flatnonzero(text[lo:e] == 10)  # noqa: PLR2004
                if nl.size:
                    cut = lo + int(nl[-1]) + 1
                elif lo == b:
                    break
                span <<= 2
            if cut > b:
                e = cut
            else:  # no newline inside the window: extend to the end of this line
                at, step = e, 1 << 16
                e = n
                while at < n:
                    nl = np.flatnonzero(text[at:at + step] == 10)  # noqa: PLR2004
                    if nl.size:
                        e = at + int(nl[0]) + 1
                        break
                    at += step
        yield b, e
        b = e


def run(argv: list[str]):  # noqa: C901, PLR0912, PLR0915
    "POST-GATK variant filtering"
    args = parse_args(argv)
    logging.basicConfig(format="%(asctime)s %(message)s", level=logging.INFO)
    logger = logging.getLogger(__name__)

    out = None
    try:
        model = None
        transformer = None
        blacklists = None

        # the CUDA context comes up on its own thread (the driver calls release the GIL) while this one unpickles the
        # model, which imports the estimator's library: the two longest start-up steps of a run side by side
        world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
        multi = world > 1
        device = args.device if args.device is not None else int(os.environ.get("LOCAL_RANK", "0"))
        numa = None
        if multi:
            from variantcalling_b200 import dist as vdist0

            numa = vdist0.bind_to_gpu_numa_node(device)
        ctx_pool = ThreadPoolExecutor(max_workers=2, thread_name_prefix="ugvc-cuda-init")
        ctx_future = ctx_pool.submit(lib.Context, device)

        def init_group():
            """The process group of a multi-rank run (NCCL on GPUs; gloo without a CUDA device, i.e. the host-emulation
            test) comes up in the background: importing torch and building the communicator take seconds, the ranks need
            it only for the SUM of the counters at the end."""
            import torch
            import torch.distributed as tdist

            if tdist.is_initialized():
                return False
            on_gpu = torch.cuda.is_available()
            tdist.init_process_group("nccl" if on_gpu else "gloo",
                                     **({"device_id": torch.device("cuda", device)} if on_gpu else {}))
            return True

        group_future = ctx_pool.submit(init_group) if multi else None
        t_start = time.perf_counter()
        startup = {}

        if args.model_file is not None:
            logger.info(f"Loading model from {args.model_file}")
            mf = _load_pickle(args.model_file)
            model = mf["xgb"]
            transformer = mf["transformer"]
        if args.blacklist is not None:
            logger.info(f"Loading blacklist from {args.blacklist}")
            blacklists = _load_pickle(args.blacklist)
        startup["pickles"] = time.perf_counter() - t_start
        if args.treat_multiallelics and args.ref_fasta is None:
            raise ValueError("Reference FASTA file is required for multiallelic treatment")
        if not os.path.exists(args.input_file):
            raise RuntimeError(f"Input file {args.input_file} does not exist")
        if not os.path.exists(args.input_file + ".tbi"):
            raise RuntimeError(f"Index file {args.input_file}.tbi does not exist")
        header = VcfHeader(bgzf_io.read_header_text(args.input_file))
        with_model = args.model_file is not None
        with_bl = args.blacklist is not None or args.blacklist_cg_insertions
        out_header = header.edited_lines(with_model=with_model, with_blacklist=with_bl)
        index, linear_index = bgzf_io.read_tbi(args.input_file + ".tbi", linear=True)
        # one process per GPU (torchrun): ranks own whole contigs, no record ever crosses ranks; the only
        # collective is the SUM of the counters at the end (NCCL on GPUs; gloo when there is no CUDA device,
        # i.e. in the host-emulation test)
        if multi:
            logger.info(f"rank {rank}: NUMA binding {numa}")
        startup["header+index"] = time.perf_counter() - t_start - startup["pickles"]
        t0 = time.perf_counter()
        ctx = ctx_future.result()  # raises without a CUDA device: there is no CPU path
        ctx_pool.shutdown(wait=False)
        startup["wait for CUDA"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        plan = None
        if with_model:
            if model is None or transformer is None:
                raise ValueError("Model and transformer must be loaded before applying classifier")
            plan = MC.compile_plan(header, transformer, model, args.custom_annotations)
        else:
            plan = MC.compile_plan_no_model(header)
        ctx.load_plan(plan.blob)
        recal = bool(args.recalibrate_genotype and with_model)
        split_sites = bool(args.treat_multiallelics and with_model)
        idx_ctx = None
        if split_sites:
            # the split rows' likelihoods are merged on the host before the phred step: K3 hands back
            # the fp64 likelihoods; a second context with the model-less plan indexes each contig first
            ctx.enable_phreds(2)
            idx_ctx = lib.Context(device)
            idx_ctx.load_plan(MC.compile_plan_no_model(header).blob)
        elif recal:
            ctx.enable_phreds(True)
        idx_reserved = (0, 0)
        batch_bytes = max(1, args.batch_mb) << 20
        n_lanes = 2
        reserved = (0, 0)
        key_order_set = False

        startup["plan"] = time.perf_counter() - t0
        out = _Splicer(_part_path(args.output_file, rank) if multi else args.output_file, args.io_threads)
        out.keep_arrays = multi
        if not multi:
            out.write_header(out_header)
        seconds = {"inflate_wait": 0.0, "gpu": 0.0, "alloc": 0.0}
        totals = {"n_records": 0, "n_low_score": 0, "n_cg": 0, "n_blacklisted": 0}

        def blacklist_codes(ri, n, bl_pos):
            """Per-record index into a table of ';'-joined blacklist annotations (merge order: CG
            insertions first, then each blacklist; blacklist.py:64-101)."""
            if not with_bl:
                return None, b"", None
            code = np.zeros(n, dtype=np.int32)
            parts = []  # (bit weight, annotation) in merge order
            w = 1
            if args.blacklist_cg_insertions:
                code += (ri["flags"] & 1).astype(np.int32) * w
                parts.append("CG_NON_HMER_INDEL")
                w *= 2
            for ann, pos in bl_pos:
                hit = np.isin(ri["pos"].astype(np.int64), pos)
                code += hit.astype(np.int32) * w
                parts.append(ann)
                w *= 2
            strings = []
            for c in range(w):
                vals = [parts[k] if (c >> k) & 1 else "PASS" for k in range(len(parts))]
                strings.append(";".join(vals).encode())
            totals["n_blacklisted"] += int(np.count_nonzero(code))
            totals["n_cg"] += int(np.count_nonzero(ri["flags"] & 1))
            return (code, b"".join(strings),
                    np.concatenate(([0], np.cumsum([len(x) for x in strings]))).astype(np.int64))

        contigs = [str(c) for c in (header.contigs.keys() if args.limit_to_contigs is None else args.limit_to_contigs)]
        all_contigs = list(contigs)
        if multi:
            from variantcalling_b200 import dist as vdist

            # load = compressed span of the contig in the input (a proxy for its record count that needs no pass)
            loads = {c: int((index[c][1] >> 16) - (index[c][0] >> 16)) + 1 for c in dict.fromkeys(contigs) if c in index}
            mine = set(vdist.lpt_partition(loads, world)[rank])
            contigs = [c for c in contigs if c in mine or (c not in index and rank == 0)]
            logger.info(f"rank {rank}/{world}: {len(contigs)} of {len(all_contigs)} contigs")

        # compressed bytes both ways: the contig's BGZF blocks go to the device as they are, come back filtered, edited
        # and compressed again (ugvc_filter_bgzf_edits: with or without a model, blacklists, --recalibrate_genotype; the
        # writer also reads INFO/END, where the index ends a record when the header declares the tag, as htslib does).
        # --treat_multiallelics takes one whole contig a call through ugvc_filter_bgzf_split (index pass, split build,
        # scored pass, merge and score math chained on the device); UGVC_MA_HOST=1 keeps it on the host readers / writers
        out.index_info_end = "END" in header.info
        split_device = bool(split_sites and not args.host_io and os.environ.get("UGVC_MA_HOST", "0") in ("", "0"))
        device_io = bool((not split_sites or split_device) and not args.host_io)
        file_flags = (lib.FILE_OVERWRITE_QUAL if args.overwrite_qual_tag else 0) | \
                     (lib.FILE_BLACKLIST_CG if args.blacklist_cg_insertions else 0)

        def load_contig(contig: str, piece: tuple | None = None):
            """Inflate one contig's records, or the piece of it between two virtual offsets (runs one contig ahead of
            the loop, on its own thread)."""
            if contig not in index:
                return None
            vb, ve = piece if piece is not None else index[contig]
            text = bgzf_io.inflate(args.input_file, vb, ve, n_threads=args.io_threads)
            if text.size == 0:
                return None
            if text[-1] != 10:  # noqa: PLR2004
                text = np.concatenate((text, np.array([10], dtype=np.uint8)))
            return text, bgzf_io.count_lines(text, args.io_threads)

        in_pool, out_pool = _PinnedPool(3), _PinnedPool(3)  # two device calls in flight + the reader / the writer
        split_plans = [None]  # --treat_multiallelics: the device split plan, carried from contig to contig
        dev_ms = np.zeros(8)  # stage ms of the device calls (5 stages of ugvc_filter_bgzf_edits, 8 of ugvc_filter_bgzf_split)

        def host_contig(contig: str, loaded):
            """One contig through the host readers / writers (text inflated on the host, records spliced on host threads)."""
            nonlocal reserved, idx_reserved, key_order_set
            text, n_contig = loaded
            logger.info(f"{n_contig} variants found on {contig}")
            if blacklists is not None:
                logger.info("Applying blacklist")
            if args.blacklist_cg_insertions:
                logger.info("Marking CG insertions")
            bl_pos = _blacklist_positions(blacklists, contig) if blacklists is not None else []

            if not key_order_set and with_model:
                head = text[: min(text.size, 1 << 20)].tobytes()
                ctx.set_key_order(*lib.learn_key_order(head[: head.rfind(b"\n") + 1]))
                key_order_set = True
            if split_sites:
                # --treat_multiallelics: the whole contig at once, like the reference's frame
                # (filter_variants_pipeline.py:145-166)
                need_idx = (text.size + 4096, n_contig + 128)
                if need_idx[0] > idx_reserved[0] or need_idx[1] > idx_reserved[1]:
                    idx_reserved = (max(need_idx[0], idx_reserved[0]), max(need_idx[1], idx_reserved[1]))
                    idx_ctx.reserve(idx_reserved[0], idx_reserved[1], n_lanes)  # (the device path's lanes too)
                idx = idx_ctx.filter_batch(text, args.decision_threshold)
                logger.info("Processing multiallelics -> pre-classifier")
                sp = split_plans[0] = multiallelics.make_split_plan(
                    header, header.loader_columns(args.custom_annotations),
                    multiallelics.read_fasta_contig(args.ref_fasta, contig, as_bytes=True), device, reuse=split_plans[0])
                scored_text = sp.build(text, idx["line_start"], idx["recinfo"])
                n_scored = getattr(sp, "n_scored_records", None)  # (the device plan counted them)
                if n_scored is None:
                    n_scored = int(np.count_nonzero(scored_text == 10))  # noqa: PLR2004
                need = (scored_text.size + 4096, n_scored + 128)
                if need[0] > reserved[0] or need[1] > reserved[1]:
                    reserved = (max(need[0], reserved[0]), max(need[1], reserved[1]))
                    ctx.reserve(reserved[0], reserved[1], n_lanes)
                scored = ctx.filter_batch(scored_text, args.decision_threshold, want_recinfo=False)
                lik = sp.merge(ctx.collect_phreds(0, scored["n_records"]))
                phreds, quals, low = multiallelics.score_math(lik, args.decision_threshold)
                n = idx["n_records"]
                res = {"n_records": n, "line_start": idx["line_start"], "recinfo": idx["recinfo"],
                       "low_score": np.ascontiguousarray(low), "qual": np.ascontiguousarray(quals)}
                bl_code, bl_table, bl_off = blacklist_codes(res["recinfo"], n, bl_pos)
                logger.info("Writing records")
                out.write_batch(contig, text, res, with_model=True, overwrite_qual=args.overwrite_qual_tag,
                                bl_code=bl_code, bl_table=bl_table, bl_off=bl_off,
                                phreds=np.ascontiguousarray(phreds) if recal else None)
                totals["n_records"] += n
                totals["n_low_score"] += int(low.sum())
                logger.info(f"{contig} done")
                return

            ranges = list(_split_batches(text, batch_bytes))
            # records per batch (one scan of the text at most: a contig that fits one batch was counted on load)
            n_in = [n_contig] if len(ranges) == 1 else [bgzf_io.count_lines(text[b:e], args.io_threads) for b, e in ranges]
            need = (max(e - b for b, e in ranges) + 4096, max(n_in) + 128)
            if need[0] > reserved[0] or need[1] > reserved[1]:
                reserved = (max(need[0], reserved[0]), max(need[1], reserved[1]))
                ctx.reserve(reserved[0], reserved[1], n_lanes)

            logger.info("Writing records")
            inflight: list[tuple[int, int, int, int]] = []

            def finish(item, contig=contig, text=text, bl_pos=bl_pos):
                lane, b, e, cap = item
                outs = ctx.alloc_outputs(cap, want_recinfo=True)
                t_gpu = time.perf_counter()
                n = ctx.collect(lane, outs, cap)
                seconds["gpu"] += time.perf_counter() - t_gpu
                res = ctx.trim_outputs(outs, n)
                phreds = np.ascontiguousarray(ctx.collect_phreds(lane, n)) if recal else None
                bl_code, bl_table, bl_off = blacklist_codes(res["recinfo"], n, bl_pos)
                out.write_batch(contig, text[b:e], res, with_model=with_model,
                                overwrite_qual=args.overwrite_qual_tag, bl_code=bl_code, bl_table=bl_table,
                                bl_off=bl_off, phreds=phreds)
                totals["n_records"] += n
                if with_model:
                    totals["n_low_score"] += int(res["low_score"].sum())

            for bi, (b, e) in enumerate(ranges):
                lane = bi % n_lanes
                if len(inflight) == n_lanes:
                    finish(inflight.pop(0))
                chunk = text[b:e]
                ctx.submit(lane, chunk, chunk.size, args.decision_threshold)
                inflight.append((lane, b, e, n_in[bi] + 1))
            while inflight:
                finish(inflight.pop(0))
            logger.info(f"{contig} done")


        # ---- work list: the host path takes a contig at a time; the device-side file path takes runs of contigs that are
        # adjacent in the file, so that a call inflates / encodes tens of thousands of BGZF blocks at once (a block is a
        # warp's work: small contigs alone leave most of the GPU idle).  Multi-rank runs keep whole contigs per call: rank 0
        # copies each contig's blocks verbatim, which needs them to start on a block boundary.
        def device_groups():
            """[[(contig, begin voff, end voff), ...], ...]: pieces adjacent in the file, about group_bytes compressed a group.
            Contigs longer than that are cut at entries of the tabix linear index (record starts).  --treat_multiallelics:
            one whole contig a group (its overlap clusters must not be cut)."""
            pieces = []
            for c in contigs:
                if c not in index:
                    continue
                vb, ve = index[c]
                cuts = [vb]
                if not multi and not split_device:
                    for v in linear_index.get(c, ()):
                        if (int(v) >> 16) - (cuts[-1] >> 16) >= group_bytes and (ve >> 16) - (int(v) >> 16) >= group_bytes // 4:
                            cuts.append(int(v))
                cuts.append(ve)
                pieces += [(c, cuts[k], cuts[k + 1]) for k in range(len(cuts) - 1)]
            groups, cur, cur_bytes = [], [], 0
            for c, vb, ve in pieces:
                span = (ve >> 16) - (vb >> 16)
                # blacklist positions are uploaded per call for one contig: with blacklists a group holds one contig
                if cur and (multi or split_device or vb != cur[-1][2] or cur_bytes + span > group_bytes + group_bytes // 4 or
                            (blacklists is not None and c != cur[-1][0])):
                    groups.append(cur)
                    cur, cur_bytes = [], 0
                cur.append((c, vb, ve))
                cur_bytes += span
            if cur:
                groups.append(cur)
            return groups

        # compressed bytes a call: about batch_mb / 2 of text at the usual ratio of 4 -- thousands of BGZF blocks in flight
        # (a block is a warp's work), buffers small enough that page-locking them does not cost more than the copies save
        group_bytes = max(1, args.batch_mb) << 17
        work = device_groups() if device_io else [[(c, 0, 0)] for c in contigs]
        max_span = max([(g[-1][2] >> 16) - (g[0][1] >> 16) + (1 << 16) for g in work], default=0) if device_io else 0
        for c in contigs if device_io else []:
            if c not in index:
                logger.info(f"Filtering variants from {c}")
                logger.info(f"No variants found on {c}")

        def load_group(group: list[tuple]):
            """The compressed blocks of a run of adjacent pieces and where each piece's text begins in them."""
            infos = [bgzf_io.range_info(args.input_file, vb, ve) for _c, vb, ve in group]
            live = [(g, i) for g, i in zip(group, infos) if i[3] > 0]
            if not live:
                return None
            c0, c1, skip = live[0][1][0], live[-1][1][1], live[0][1][2]
            starts, take = [], 0
            for _g, i in live:
                starts.append(take)
                take += i[3]
            ctx.bind_thread()  # the reader thread pins memory for this rank's device
            bufs = in_pool.acquire({"comp": (c1 - c0, np.uint8)}, grow=max_span / max(1, c1 - c0))
            comp = bufs["comp"][1]
            with open(args.input_file, "rb") as fh:
                fh.seek(c0)
                got = fh.readinto(memoryview(comp))
            if got != c1 - c0:
                raise OSError(f"{args.input_file}: short read of {group[0][0]}..{group[-1][0]}")
            ref = multiallelics.read_fasta_contig(args.ref_fasta, group[0][0], as_bytes=True) if split_device else None
            return "device", comp, skip, take, bufs, [g for g, _ in live], np.array(starts, dtype=np.uint64), ref

        def load_work(group: list[tuple]):
            return load_group(group) if device_io else load_contig(group[0][0])

        # device-side file path: two calls in flight (one lane and stream each, issued from two host threads), so that one
        # piece's copies and host-side waits overlap the other's kernels; results are written in submission order
        gpu_pool = ThreadPoolExecutor(max_workers=n_lanes, thread_name_prefix="ugvc-device")
        flying: list[tuple] = []
        n_calls = 0
        # --treat_multiallelics on the device: a split handle per lane (a handle serves one stream at a time)
        lane_plans = [multiallelics.DeviceSplitPlan(header, header.loader_columns(args.custom_annotations), b"", device)
                      for _ in range(n_lanes)] if split_device else []

        def device_call(lane: int, comp, skip: int, take: int, in_bufs: dict, starts, bl_pos, ref):
            ctx.bind_thread()
            n_max = take // 32 + 1024
            # VCF text deflates to well under half its size; text that does not comes back as UGVC_E_FALLBACK
            sizes = {"out": (take * 5 // 8 + (1 << 20), np.uint8), "blocks": ((take + n_max * 64) // lib.DEF_CHUNK + 16, np.uint32),
                     "ri": (n_max, lib.RECINFO_DTYPE), "ls": (n_max + 1, np.int64), "low": (n_max, np.uint8)}
            if out.index_info_end:
                sizes["end"] = (n_max, np.int64)
            out_bufs = out_pool.acquire(sizes, grow=max_span / max(1, comp.size))
            try:
                if split_device:
                    sp = lane_plans[lane]
                    sp.set_reference(ref)
                    res = sp.filter_bgzf(ctx, idx_ctx, comp, skip, take, args.decision_threshold, file_flags, n_max,
                                         recalibrate_genotype=recal, blacklists=bl_pos, want_end=out.index_info_end, lane=lane,
                                         bufs={k: v[1] for k, v in out_bufs.items()})
                    first = np.zeros(1, dtype=np.int64) if res is not None else None
                    ms = ctx.filter_bgzf_split_stage_ms(lane) if res is not None else None
                else:
                    res = ctx.filter_bgzf_edits(comp, skip, take, args.decision_threshold, file_flags, n_max, with_model=with_model,
                                                recalibrate_genotype=recal, blacklists=bl_pos, want_end=out.index_info_end,
                                                lane=lane, bufs={k: v[1] for k, v in out_bufs.items()})
                    first = ctx.filter_bgzf_first_records(starts, lane=lane) if res is not None else None
                    ms = ctx.filter_bgzf_stage_ms(lane) if res is not None else None
            except BaseException:
                out_pool.release(out_bufs)
                raise
            finally:
                in_pool.release(in_bufs)
            if res is None:
                out_pool.release(out_bufs)
            return res, first, ms, out_bufs

        def drain_device(leave: int):
            """Take finished device calls (oldest first) until `leave` are in flight; write their records."""
            nonlocal dev_ms
            while len(flying) > leave:
                live, fut = flying.pop(0)
                t_gpu = time.perf_counter()
                res, first, ms, out_bufs = fut.result()
                seconds["gpu"] += time.perf_counter() - t_gpu
                if res is None:
                    logger.info(f"{live[0][0]}..{live[-1][0]}: records that need the general writer, taking the host path")
                    for _l, f in flying:
                        f.exception()  # the host path uses the same lanes: newer calls finish first (written after these records)
                    for c, vb, ve in live:
                        again = load_contig(c, (vb, ve))
                        if again is not None:
                            host_contig(c, again)
                    continue
                dev_ms[: len(ms)] += np.array(ms)
                bounds = np.concatenate((first, [res["n_records"]])).astype(np.int64)
                for k, (c, _vb, _ve) in enumerate(live):
                    logger.info(f"{int(bounds[k + 1] - bounds[k])} variants found on {c}")
                if split_device:
                    logger.info("Processing multiallelics -> pre-classifier")
                logger.info("Writing records")
                out.write_device_batch([g[0] for g in live], bounds, res, release=lambda b=out_bufs: out_pool.release(b))
                totals["n_records"] += res["n_records"]
                if with_model:
                    totals["n_low_score"] += int(res["low_score"].sum())
                if with_bl:  # what blacklist_codes counts on the host path
                    totals["n_cg"] += int(np.count_nonzero(res["recinfo"]["flags"] & 1))
                    totals["n_blacklisted"] += res["n_blacklisted"]
                for c in dict.fromkeys(g[0] for g in live):
                    logger.info(f"{c} done")

        prefetch = ThreadPoolExecutor(max_workers=1, thread_name_prefix="ugvc-bgzf-reader")
        bl_last = [None, None]  # (contig, its blacklist positions) of the last device group
        pending = prefetch.submit(load_work, work[0]) if work else None
        for gi, group in enumerate(work):
            for c in dict.fromkeys(g[0] for g in group):
                logger.info(f"Filtering variants from {c}")
            t_wait = time.perf_counter()
            loaded = pending.result()
            seconds["inflate_wait"] += time.perf_counter() - t_wait
            pending = prefetch.submit(load_work, work[gi + 1]) if gi + 1 < len(work) else None
            if loaded is None:
                for c in dict.fromkeys(g[0] for g in group):
                    logger.info(f"No variants found on {c}")
                continue
            if not isinstance(loaded[0], str):
                host_contig(group[0][0], loaded)
                continue
            _tag, comp, skip, take, in_bufs, live, starts, ref = loaded  # ("device", compressed blocks, ...)
            if blacklists is not None:
                logger.info("Applying blacklist")
            if args.blacklist_cg_insertions:
                logger.info("Marking CG insertions")
            bl_pos = None
            if blacklists is not None:  # (one contig a group) a long contig is many groups: its positions are kept
                if bl_last[0] != live[0][0]:
                    bl_last[:] = [live[0][0], _blacklist_positions(blacklists, live[0][0])]
                bl_pos = bl_last[1]
            if not key_order_set and with_model:
                head = bgzf_io.first_block_text(comp, skip)
                ctx.set_key_order(*lib.learn_key_order(head[: head.rfind(b"\n") + 1]))
                key_order_set = True
            need = (take + (1 << 17) + 4096, take // 32 + 1024)  # whole blocks are inflated: up to 64 KiB either side of the range
            # --treat_multiallelics: the index pass reads the contig, the scored pass the kept lines and up to two split rows
            # for every record taken out (a contig that outgrows this comes back as a fall-back)
            need_idx, need = (need, (2 * need[0], 2 * need[1])) if split_device else (None, need)
            t_alloc = time.perf_counter()
            if need[0] > reserved[0] or need[1] > reserved[1] or \
                    (need_idx and (need_idx[0] > idx_reserved[0] or need_idx[1] > idx_reserved[1])):
                drain_device(0)  # the lanes' buffers are about to move
                ahead = max(1.0, max_span / max(1, comp.size)) * 1.05  # the largest group, at this one's compression ratio
                if need[0] > reserved[0] or need[1] > reserved[1]:
                    reserved = (max(int(need[0] * ahead), reserved[0]), max(int(need[1] * ahead), reserved[1]))
                    ctx.reserve(reserved[0], reserved[1], n_lanes)
                if need_idx and (need_idx[0] > idx_reserved[0] or need_idx[1] > idx_reserved[1]):
                    idx_reserved = (max(int(need_idx[0] * ahead), idx_reserved[0]), max(int(need_idx[1] * ahead), idx_reserved[1]))
                    idx_ctx.reserve(idx_reserved[0], idx_reserved[1], n_lanes)
            seconds["alloc"] += time.perf_counter() - t_alloc
            drain_device(n_lanes - 1)  # at most n_lanes calls in flight, each on its own lane and stream
            flying.append((live, gpu_pool.submit(device_call, n_calls % n_lanes, comp, skip, take, in_bufs, starts, bl_pos, ref)))
            n_calls += 1
            if n_calls == 1:
                drain_device(0)  # the first call alone: every lazy one-time set-up of the path happens on one thread
        drain_device(0)
        gpu_pool.shutdown()

        t_close = time.perf_counter()
        if multi:
            import torch
            import torch.distributed as tdist

            with open(_part_path(args.output_file, rank) + ".meta", "wb") as fh:
                pickle.dump(out.finish_part(), fh)
            created_group = group_future.result()
            keys = ("n_records", "n_low_score", "n_cg", "n_blacklisted")
            counts = torch.tensor([totals[k] for k in keys], dtype=torch.int64,
                                  device=torch.device("cuda", device) if torch.cuda.is_available() else "cpu")
            vdist.allreduce_counts(counts)  # the single collective of the path; it also orders the parts before rank 0 reads them
            totals.update({k: int(v) for k, v in zip(keys, counts.tolist())})
            if rank == 0:
                t_asm = time.perf_counter()
                _assemble_parts(args.output_file, out_header, all_contigs, world, args.io_threads)
                logger.info("parts assembled and indexed in %.2f s", time.perf_counter() - t_asm)
            tdist.barrier()
            if created_group:
                tdist.destroy_process_group()
        else:
            out.close(args.output_file)
        prefetch.shutdown()
        logger.info("stage seconds (overlapping threads): wait for inflate %.2f, buffers %.2f, wait for GPU %.2f, splice %.2f, "
                    "deflate+write %.2f, index %.2f (+ %.2f at close)", seconds["inflate_wait"], seconds["alloc"], seconds["gpu"],
                    out.seconds["splice"], out.seconds["deflate"], out.seconds.get("index", 0.0), time.perf_counter() - t_close)
        logger.info("start-up seconds: " + ", ".join(f"{k} {v:.2f}" for k, v in startup.items()))
        if split_device:
            logger.info("device split path, ms on the GPU: H2D + inflate %.0f, index K1 %.0f, split build %.0f, scored K1..K3 %.0f, "
                        "merge + score %.0f, record writer %.0f, deflate + pack %.0f, D2H %.0f", *dev_ms)
        elif device_io:
            logger.info("device file path, ms on the GPU: H2D + inflate %.0f, K1..K3 %.0f, record writer %.0f, deflate + pack %.0f, "
                        "D2H %.0f", *dev_ms[:5])
        ctx.close()
        for sp in lane_plans:
            sp.close()
        if idx_ctx is not None:
            idx_ctx.close()
        if split_plans[0] is not None and hasattr(split_plans[0], "close"):
            split_plans[0].close()
        logger.info(
            f"{totals['n_records']} records written: {totals['n_low_score']} LOW_SCORE, "
            f"{totals['n_records'] - totals['n_low_score']} not LOW_SCORE, {totals['n_blacklisted']} blacklisted")
        logger.info("Variant filtering run: success")
        return totals

    except Exception as err:
        if out is not None:
            out.abort()
        exc_info = sys.exc_info()
        logger.error(exc_info[:2])
        logger.exception(err)
        logger.error("Variant filtering run: failed")
        raise err


def main():
    run(sys.argv[1:])


if __name__ == "__main__":
    main()
