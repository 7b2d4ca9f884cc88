"""The device file path shared by the VCF tools (``low_af_ratio.py``, ``bridging_snvs.py``, ``gvcf_hcr.py``; DESIGN.md
4c, 4d, 4e).

The input (BGZF or plain text) is cut into pieces of whole lines of about ``piece_bytes`` of text, each piece is one
device call, two pieces are in flight on two lanes, and the ``.tbi`` of the written records is built from the virtual
offsets of the device-written blocks (htslib's rules: DESIGN.md 4).
"""
from __future__ import annotations

import os
import struct
import threading
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from variantcalling_b200 import bgzf_io, lib


def blocks(raw: np.ndarray) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Compressed offset, compressed size and uncompressed size of every BGZF block of a file's bytes."""
    mv = memoryview(raw)
    coff, csz, usz = [], [], []
    at, n = 0, raw.size
    while at < n:
        if n - at < 28 or mv[at] != 0x1F or mv[at + 1] != 0x8B:
            raise OSError(f"not a BGZF block at byte {at}")
        xlen = struct.unpack_from("<H", mv, at + 10)[0]
        bsize, x = None, at + 12
        while x < at + 12 + xlen:
            si1, si2, slen = struct.unpack_from("<BBH", mv, x)
            if (si1, si2, slen) == (66, 67, 2):
                bsize = struct.unpack_from("<H", mv, x + 4)[0] + 1
            x += 4 + slen
        if bsize is None or at + bsize > n:
            raise OSError(f"bad BGZF block at byte {at}")
        coff.append(at)
        csz.append(bsize)
        usz.append(struct.unpack_from("<I", mv, at + bsize - 4)[0])
        at += bsize
    return np.array(coff, np.int64), np.array(csz, np.int64), np.array(usz, np.int64)


def inflate_block(raw: np.ndarray, coff: int, csize: int) -> bytes:
    xlen = struct.unpack_from("<H", memoryview(raw), coff + 10)[0]
    return zlib.decompress(bytes(raw[coff + 12 + xlen: coff + csize - 8]), -15)


def bgzf_cuts(path: str, raw: np.ndarray, coff, csz, ustart, data_begin: int, total: int, piece_bytes: int,
              index_cuts: bool = True) -> list[int]:
    """Uncompressed offsets where pieces begin (line starts), about piece_bytes apart: from the .tbi linear index when
    there is one (and index_cuts), else at the first line start of a block (that block inflated on the host)."""
    cuts = [data_begin]
    cands: list[int] = []
    if index_cuts and os.path.exists(path + ".tbi"):
        try:
            _, lin = bgzf_io.read_tbi(path + ".tbi", linear=True)
            voffs = np.unique(np.concatenate([v for v in lin.values()] or [np.zeros(0, np.uint64)]))
            blk = np.searchsorted(coff, (voffs >> np.uint64(16)).astype(np.int64))
            ok = (blk < coff.size) & (coff[np.minimum(blk, coff.size - 1)] == (voffs >> np.uint64(16)).astype(np.int64))
            cands = sorted(int(ustart[b] + (v & np.uint64(0xFFFF))) for b, v in zip(blk[ok], voffs[ok]))
        except OSError:
            cands = []
    if cands:
        for u in cands:
            if u - cuts[-1] >= piece_bytes and u < total:
                cuts.append(u)
    else:
        b = int(np.searchsorted(ustart, cuts[-1] + piece_bytes))
        while b < coff.size and ustart[b] < total:
            nl = inflate_block(raw, int(coff[b]), int(csz[b])).find(b"\n")
            if nl >= 0 and ustart[b] + nl + 1 < total:
                cuts.append(int(ustart[b]) + nl + 1)
                b = int(np.searchsorted(ustart, cuts[-1] + piece_bytes))
            else:  # a line longer than the block: the next block
                b += 1
    return cuts + [total]


def text_cuts(text: np.ndarray, data_begin: int, piece_bytes: int) -> list[int]:
    cuts = [data_begin]
    while text.size - cuts[-1] > piece_bytes:
        nl = np.flatnonzero(text[cuts[-1] + piece_bytes:] == 10)  # noqa: PLR2004
        if not nl.size or cuts[-1] + piece_bytes + int(nl[0]) + 1 >= text.size:
            break
        cuts.append(cuts[-1] + piece_bytes + int(nl[0]) + 1)
    return [*cuts, text.size]


class Input:
    """A VCF file cut into pieces of whole data lines: ``pieces[k] = (data, skip_head, take_bytes, span)`` as the device
    calls take them, ``starts[k]`` the uncompressed offset of piece k's first line.  index_cuts=False cuts a BGZF file at
    block line starts even when it has a ``.tbi``, so that pieces follow piece_bytes whatever the records' density."""

    def __init__(self, path: str, data_begin: int, piece_bytes: int, index_cuts: bool = True):
        self.path = path
        raw = np.fromfile(path, dtype=np.uint8)
        self.raw = raw
        self.is_bgzf = raw.size >= 2 and raw[0] == 0x1F and raw[1] == 0x8B  # noqa: PLR2004
        if self.is_bgzf:
            self.coff, self.csz, usz = blocks(raw)
            self.ustart = np.concatenate(([0], np.cumsum(usz)))
            total = int(self.ustart[-1])
            cuts = bgzf_cuts(path, raw, self.coff, self.csz, self.ustart[:-1], data_begin, total, piece_bytes, index_cuts)
        else:
            cuts = text_cuts(raw, data_begin, piece_bytes)
        self.pieces, self.starts = [], []
        for u0, u1 in zip(cuts[:-1], cuts[1:]):
            if u1 <= u0:
                continue
            if self.is_bgzf:
                b0 = int(np.searchsorted(self.ustart, u0, side="right")) - 1
                b1 = int(np.searchsorted(self.ustart, u1 - 1, side="right")) - 1
                span = int(self.ustart[b1 + 1] - self.ustart[b0])
                self.pieces.append((raw[self.coff[b0]: self.coff[b1] + self.csz[b1]], u0 - int(self.ustart[b0]), u1 - u0, span))
            else:
                self.pieces.append((raw[u0:u1], 0, u1 - u0, u1 - u0))
            self.starts.append(u0)
        if self.pieces and not self.is_bgzf and raw[cuts[-1] - 1] != 10:  # noqa: PLR2004
            raise ValueError(f"{path}: the last line has no newline")
        self._cache: tuple[int, bytes] = (-1, b"")

    def text(self, u0: int, u1: int) -> bytes:
        """Uncompressed bytes [u0, u1) of the input, clipped at its end (BGZF blocks inflated on the host, the last one
        kept)."""
        if not self.is_bgzf:
            return self.raw[u0:u1].tobytes()
        out = []
        b = int(np.searchsorted(self.ustart, u0, side="right")) - 1
        while u0 < u1 and b < self.coff.size:
            cached = self._cache  # read once: the calls of the other lane's thread may replace it
            if cached[0] != b:
                cached = (b, inflate_block(self.raw, int(self.coff[b]), int(self.csz[b])))
                self._cache = cached
            blk = cached[1]
            lo = u0 - int(self.ustart[b])
            take = min(len(blk) - lo, u1 - u0)
            out.append(blk[lo: lo + take])
            u0 += take
            b += 1
        return b"".join(out)

    def line_at(self, u0: int, r: int) -> str:
        """Data line r of the piece that starts at uncompressed offset u0 (read back from the input)."""
        at, chunk = u0, b""
        for _ in range(r + 1):
            at += len(chunk)
            chunk = self.text(at, at + (1 << 16))
            while b"\n" not in chunk:
                more = self.text(at + len(chunk), at + len(chunk) + (1 << 16))
                if not more:
                    break
                chunk += more
            chunk = chunk[: chunk.find(b"\n") + 1] if b"\n" in chunk else chunk
        return chunk.rstrip(b"\n").decode("latin-1")


def run_on_lanes(ctx: lib.Context, n_pieces: int, call, thread_name: str):
    """Yield (k, call(k, lane)) for k = 0 .. n_pieces - 1 in order, with up to two calls in flight on two lanes (the
    context reserved with that many lanes).  An exception of call(k, ...) is raised when piece k's turn comes.  Close the
    generator (contextlib.closing) so that no call is still running when the caller frees the context."""
    n_lanes = 2 if n_pieces > 1 else 1
    locks = [threading.Lock() for _ in range(n_lanes)]

    def one(k: int):
        with locks[k % n_lanes]:
            return call(k, k % n_lanes)

    with ThreadPoolExecutor(max_workers=n_lanes, thread_name_prefix=thread_name) as pool:
        futures = [pool.submit(one, k) for k in range(n_pieces)]
        for k, fut in enumerate(futures):
            yield k, fut.result()


class Index:
    """Contig runs and tabix intervals of the written records (htslib's rules: DESIGN.md 4).  A call's result carries
    ``flags`` whose bit ``lib.AFR_NEW_CONTIG`` marks the first record of each contig run."""

    def __init__(self, info_end: bool):
        self.info_end = info_end
        self.names: list[str] = []
        self.cur: list[tuple] = []
        self.sections: list[bytes] = []
        self.last_pos = -1

    def add(self, writer: bgzf_io.BgzfWriter, res: dict, base: int):
        n = res["n_records"]
        if n == 0:
            return
        ri, ls = res["recinfo"], res["line_start"]
        beg = ri["pos"].astype(np.int64) - 1
        end = beg + np.maximum(1, (ri["flags"] >> 8).astype(np.int64))
        if self.info_end:
            end = np.where(res["end"] > beg, res["end"], end)
        vs = writer.virtual_offsets(base + ls[:-1])
        ve = writer.virtual_offsets(base + ls[1:] - 1) + np.uint64(1)
        starts = np.flatnonzero(res["flags"] & lib.AFR_NEW_CONTIG)
        bounds = [*starts.tolist(), n]
        for k, r0 in enumerate(starts.tolist()):
            r1 = bounds[k + 1]
            name = self._name(res, r0)
            if not self.names or self.names[-1] != name:
                if name in self.names:
                    raise ValueError(f"records of contig {name} are not contiguous: the output cannot be indexed")
                self._close()
                self.names.append(name)
                self.last_pos = -1
            b = beg[r0:r1]
            if b[0] < self.last_pos or np.any(b[1:] < b[:-1]):
                raise ValueError(f"records of contig {name} are not sorted by position: the output cannot be indexed")
            self.last_pos = int(b[-1])
            self.cur.append((b, end[r0:r1], vs[r0:r1], ve[r0:r1]))

    @staticmethod
    def _name(res: dict, r: int) -> str:
        """CHROM of record r, read back from the call's output blocks (contig runs are few)."""
        off = int(res["line_start"][r])
        cs = res["block_csize"].astype(np.int64)
        cstart = np.concatenate(([0], np.cumsum(cs)))
        k = off // lib.DEF_CHUNK
        buf = b""
        while k < cs.size:
            buf += inflate_block(res["bgzf"], int(cstart[k]), int(cs[k]))
            tab = buf.find(b"\t", off - (off // lib.DEF_CHUNK) * lib.DEF_CHUNK)
            if tab >= 0:
                return buf[off - (off // lib.DEF_CHUNK) * lib.DEF_CHUNK: tab].decode()
            k += 1
        raise ValueError(f"record {r} has a single column")

    def _close(self):
        if self.names:
            cols = [np.concatenate([c[k] for c in self.cur]) for k in range(4)] if self.cur else [np.zeros(0, np.int64)] * 4
            self.sections.append(bgzf_io.tbi_section(cols[0], cols[1], cols[2].astype(np.uint64), cols[3].astype(np.uint64)))
        self.cur = []

    def write(self, path: str):
        self._close()
        bgzf_io.write_tbi(path, bgzf_io.tbi_assemble(self.names, self.sections))
