"""DEFLATE streams written by hand (RFC 1951) inside BGZF blocks (SAM spec 4.1), for testing decoders at shapes zlib's
own encoder never emits: explicit code lengths, long codes, chosen code-length repeats, explicit length / distance
symbols, stored blocks at any bit offset, and streams that are wrong in exactly one way.

A block is written into a :class:`BitWriter` by :func:`stored`, :func:`fixed` or :func:`dynamic` from a token list:
an ``int`` below 256 is a literal, :class:`Match` a (length, distance) pair, :class:`Sym` / :class:`DSym` /
:class:`Bits` raw literal-length symbols, distance symbols and bits (for streams that must be invalid).  The
end-of-block code is appended unless ``eob=False``.  :func:`bgzf_block` wraps a payload; ISIZE and CRC default to
those of the intended output and can be overridden."""
import struct
import zlib
from dataclasses import dataclass

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32
EOB = 256


@dataclass(frozen=True)
class Match:
    """A match; ``lsym`` forces the length symbol (e.g. 284 for 258), its extra bits are length - base."""
    length: int
    dist: int
    lsym: int | None = None


@dataclass(frozen=True)
class Sym:
    """A literal-length symbol written without extra bits."""
    sym: int


@dataclass(frozen=True)
class DSym:
    """A distance symbol written without extra bits."""
    sym: int


@dataclass(frozen=True)
class Bits:
    value: int
    n: int


class BitWriter:
    """LSB-first bit writer (RFC 1951 3.1.1)."""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, value: int, n: int):
        assert 0 <= value < (1 << n) or (n == 0 and value == 0), (value, n)
        self.acc |= value << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def put_code(self, code: int, n: int):
        """A Huffman code, most significant bit first."""
        self.put(int(format(code, f"0{n}b")[::-1], 2) if n else 0, n)

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def put_bytes(self, data: bytes):
        assert self.n == 0
        self.out += data

    @property
    def bit_len(self) -> int:
        return 8 * len(self.out) + self.n

    def getvalue(self) -> bytes:
        tail = bytes([self.acc]) if self.n else b""
        return bytes(self.out) + tail


def canonical(lengths) -> dict:
    """symbol -> (code, length) of the canonical code with these lengths (RFC 1951 3.2.2); no validity check."""
    max_len = max(lengths, default=0)
    bl_count = [0] * (max_len + 2)
    for n in lengths:
        if n:
            bl_count[n] += 1
    code, next_code = 0, [0] * (max_len + 2)
    for bits in range(1, max_len + 1):
        code = (code + bl_count[bits - 1]) << 1
        next_code[bits] = code
    out = {}
    for s, n in enumerate(lengths):
        if n:
            out[s] = (next_code[n], n)
            next_code[n] += 1
    return out


def kraft(lengths) -> float:
    return sum(2.0 ** -n for n in lengths if n)


def complete_lengths(symbols, n: int) -> list[int]:
    """Code lengths over n symbols that give `symbols` (two or more) a complete, nearly flat code."""
    symbols = sorted(set(symbols))
    k = len(symbols)
    assert k >= 2  # noqa: PLR2004
    top = (k - 1).bit_length()
    n_short = (1 << top) - k                     # these get top - 1 bits, the rest top bits: Kraft sum 1
    lens = [0] * n
    for i, s in enumerate(symbols):
        lens[s] = top - 1 if i < n_short else top
    return lens


def skewed_lengths(symbols, n: int) -> list[int]:
    """A complete code with lengths 1, 2, ..., k-1, k-1 over `symbols` in the order given: 16 symbols reach 15 bits."""
    lens = [0] * n
    k = len(symbols)
    for i, s in enumerate(symbols):
        lens[s] = min(i + 1, k - 1)
    assert kraft(lens) == 1.0
    return lens


def length_symbol(length: int, lsym: int | None = None) -> tuple[int, int, int]:
    """(symbol, extra value, extra bits) of a match length."""
    if lsym is None:
        lsym = 285 if length == 258 else 257 + max(i for i in range(28) if LEN_BASE[i] <= length)  # noqa: PLR2004
    i = lsym - 257
    extra = length - LEN_BASE[i]
    assert 0 <= extra < (1 << LEN_EXTRA[i]) or (extra == 0 and LEN_EXTRA[i] == 0), (length, lsym)
    return lsym, extra, LEN_EXTRA[i]


def dist_symbol(dist: int) -> tuple[int, int, int]:
    i = max(j for j in range(30) if DIST_BASE[j] <= dist)
    return i, dist - DIST_BASE[i], DIST_EXTRA[i]


def expand(tokens, history: bytes = b"") -> bytes:
    """The bytes a token list stands for, after `history` (earlier blocks of the same stream)."""
    out = bytearray(history)
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
        elif isinstance(t, Match):
            assert 1 <= t.dist <= len(out), t
            for _ in range(t.length):
                out.append(out[-t.dist])
        else:
            raise ValueError(f"{t!r} stands for no bytes")
    return bytes(out[len(history):])


def _header(w: BitWriter, final: bool, btype: int):
    w.put(int(final), 1)
    w.put(btype, 2)


def _tokens(w: BitWriter, tokens, lit: dict, dist: dict, eob: bool):
    for t in list(tokens) + ([EOB] if eob else []):
        if isinstance(t, int):
            w.put_code(*lit[t])
        elif isinstance(t, Match):
            s, x, nx = length_symbol(t.length, t.lsym)
            w.put_code(*lit[s])
            w.put(x, nx)
            ds, dx, ndx = dist_symbol(t.dist)
            w.put_code(*dist[ds])
            w.put(dx, ndx)
        elif isinstance(t, Sym):
            w.put_code(*lit[t.sym])
        elif isinstance(t, DSym):
            w.put_code(*dist[t.sym])
        elif isinstance(t, Bits):
            w.put(t.value, t.n)
        else:
            raise TypeError(t)


def stored(w: BitWriter, data: bytes, final: bool = True, nlen: int | None = None, length: int | None = None):
    """A stored block; `length` / `nlen` override LEN / NLEN."""
    _header(w, final, 0)
    w.align()
    n = len(data) if length is None else length
    w.put(n, 16)
    w.put((~n & 0xFFFF) if nlen is None else nlen, 16)
    w.put_bytes(data)


def fixed(w: BitWriter, tokens, final: bool = True, eob: bool = True):
    _header(w, final, 1)
    _tokens(w, tokens, canonical(FIXED_LIT), canonical(FIXED_DIST), eob)


def rle_lengths(lengths) -> list[tuple[int, int]]:
    """Code-length symbols (symbol, extra value) for a sequence of lengths: 16 / 17 / 18 for runs, as zlib does."""
    out, i, n = [], 0, len(lengths)
    while i < n:
        v, r = lengths[i], 1
        while i + r < n and lengths[i + r] == v:
            r += 1
        if v == 0 and r >= 11:  # noqa: PLR2004
            k = min(r, 138)
            out.append((18, k - 11))
        elif v == 0 and r >= 3:  # noqa: PLR2004
            k = min(r, 10)
            out.append((17, k - 3))
        elif v != 0 and r >= 4:  # noqa: PLR2004
            out.append((v, 0))
            k = min(r - 1, 6)
            out.append((16, k - 3))
            k += 1
        else:
            out.append((v, 0))
            k = 1
        i += k
    return out


def dynamic(w: BitWriter, lit_lens, dist_lens, tokens, final: bool = True, eob: bool = True, cl_symbols=None,
            cl_lens=None, hlit: int | None = None, hdist: int | None = None, hclen: int | None = None):
    """A dynamic block.  lit_lens / dist_lens give HLIT / HDIST (unless overridden: the 5-bit fields are written as given
    minus 257 / 1).  cl_symbols: the code-length sequence as (symbol, extra) pairs (default: rle_lengths of the
    concatenated lengths); cl_lens: the code-length code (default: complete over the symbols used); hclen: how many
    code-length code lengths are written (default: up to the last non-zero in CL_ORDER, at least 4)."""
    lit_lens, dist_lens = list(lit_lens), list(dist_lens)
    hlit = len(lit_lens) if hlit is None else hlit
    hdist = len(dist_lens) if hdist is None else hdist
    if cl_symbols is None:
        cl_symbols = rle_lengths(lit_lens + dist_lens)
    if cl_lens is None:
        used = {s for s, _ in cl_symbols}
        if len(used) == 1:
            used.add(0 if 0 not in used else 1)
        cl_lens = complete_lengths(used, 19)
    if hclen is None:
        hclen = max([4] + [i + 1 for i, s in enumerate(CL_ORDER) if cl_lens[s]])
    _header(w, final, 2)
    w.put(hlit - 257, 5)
    w.put(hdist - 1, 5)
    w.put(hclen - 4, 4)
    for i in range(hclen):
        w.put(cl_lens[CL_ORDER[i]], 3)
    clc = canonical(cl_lens)
    for s, x in cl_symbols:
        w.put_code(*clc[s])
        if s == 16:  # noqa: PLR2004
            w.put(x, 2)
        elif s == 17:  # noqa: PLR2004
            w.put(x, 3)
        elif s == 18:  # noqa: PLR2004
            w.put(x, 7)
    _tokens(w, tokens, canonical(lit_lens), canonical(dist_lens), eob)


def dynamic_for(tokens, final: bool = True, history: bytes = b"", w: BitWriter | None = None) -> BitWriter:
    """A dynamic block with a complete, flat code over exactly the symbols the tokens use."""
    w = BitWriter() if w is None else w
    lits, dists = {EOB}, set()
    for t in tokens:
        if isinstance(t, int):
            lits.add(t)
        else:
            lits.add(length_symbol(t.length, t.lsym)[0])
            dists.add(dist_symbol(t.dist)[0])
    if len(lits) == 1:
        lits.add(0)
    if len(dists) == 1:
        dists.add(0 if 0 not in dists else 1)
    lit_lens = complete_lengths(lits, max(257, max(lits) + 1))
    dist_lens = complete_lengths(dists, max(dists) + 1) if dists else [0]
    dynamic(w, lit_lens, dist_lens, tokens, final)
    return w


def bgzf_block(payload: bytes, data: bytes = b"", isize: int | None = None, crc: int | None = None) -> bytes:
    """One BGZF block around a raw DEFLATE payload; ISIZE and CRC32 default to those of `data`."""
    bsize = 18 + len(payload) + 8
    assert bsize <= 65536, bsize  # noqa: PLR2004
    isize = len(data) if isize is None else isize
    crc = zlib.crc32(data) & 0xFFFFFFFF if crc is None else crc
    return (b"\x1f\x8b\x08\x04" + b"\0" * 6 + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, bsize - 1) + payload
            + struct.pack("<II", crc, isize))


def split_bgzf(data: bytes) -> list[tuple[bytes, int, int]]:
    """(payload, crc, isize) of every block of consecutive BGZF blocks written by bgzf_block."""
    out, at = [], 0
    while at < len(data):
        bsize = struct.unpack_from("<H", data, at + 16)[0] + 1
        crc, isize = struct.unpack_from("<II", data, at + bsize - 8)
        out.append((data[at + 18:at + bsize - 8], crc, isize))
        at += bsize
    return out


def host_rule(payload: bytes, isize: int, crc: int) -> bytes | None:
    """What the host BGZF reader (hostio.cpp: inflate_block, htslib's rule) makes of a block: the output, or None when
    it refuses it.  zlib must reach the end of the stream inside the payload (bytes after it are ignored), the output
    must be ISIZE bytes and its CRC32 the footer's."""
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(payload, isize + 1)
    except zlib.error:
        return None
    if not d.eof or len(out) != isize or (zlib.crc32(out) & 0xFFFFFFFF) != crc:
        return None
    return out


def zlib_error(payload: bytes) -> str | None:
    """zlib's message for a raw stream it refuses, None when it inflates to the end."""
    d = zlib.decompressobj(-15)
    try:
        d.decompress(payload)
    except zlib.error as e:
        return str(e)
    return None if d.eof else "incomplete"
