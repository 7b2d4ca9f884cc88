"""GPU: the last kernels of the device file path (csrc/fileio.cu) against exact references, at their edges.

- fio_format_g, the writer's "%g" of TREE_SCORE / QUAL, against CPython's "%g" (correctly rounded, round-half-even on
  the binary value): every six-digit tie in [1e-4, 1e6) with its neighbours, the floats around each power of ten and
  each carry into a seventh digit, random bit patterns, one whole binade, and the values the writer hands back.
- The BGZF encoder of ugvc_filter_bgzf (both deflate kernels, block offsets, pack) on inputs the writer's text never
  holds: the stored fallback, 9-bit literals, runs and short periods, matches at distance 32768 and one beyond, and
  lengths around the window and block sizes.  Every block is inflated by zlib and compared byte for byte with the
  host function that restates its kernel.
- ugvc_filter_bgzf_first_records against a lower bound (np.searchsorted) on the line starts.
"""
import ctypes as C
import gzip
import struct
import zlib

import numpy as np
import pytest

from tests import util
from variantcalling_b200 import bgzf_io, lib
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader

pytestmark = pytest.mark.gpu

CHUNK = lib.DEF_CHUNK
F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------
# "%g"
# ---------------------------------------------------------------------------------------------------------------
def _bits(x) -> int:
    return int(np.array(x, F32).view(np.uint32))


def _window(center, half: int) -> np.ndarray:
    """Every float32 within +-half ulps of `center` (positive, finite)."""
    b = _bits(center)
    return np.arange(b - half, b + half + 1, dtype=np.uint32).view(F32)


def _ulp_neighbours(v: np.ndarray) -> np.ndarray:
    return np.concatenate([np.nextafter(v, F32(-np.inf)), v, np.nextafter(v, F32(np.inf))])


def ties() -> np.ndarray:
    """Every float32 in [1e-4, 1e6) halfway between two six-digit decimals: in decade X (v in [10^X, 10^(X+1))) the
    ties are (k + 1/2) 10^(X-5), and those are binary fractions iff they equal a / 2^(6-X) with a odd."""
    def ceil_scaled(e, den):  # ceil(10^e * den), exactly
        return 10 ** e * den if e >= 0 else -(-den // 10 ** -e)

    out = []
    for X in range(-4, 6):
        den = 2 ** (6 - X)
        a = np.arange(ceil_scaled(X, den) | 1, ceil_scaled(X + 1, den), 2, dtype=np.int64)
        v = a.astype(np.float64) / den
        assert np.array_equal(v.astype(F32).astype(np.float64), v)  # exact in float32 (a < 2^24)
        assert (v >= 10.0 ** X).all() and (v < 10.0 ** (X + 1)).all()
        out.append(v.astype(F32))
    return np.concatenate(out)


def expected_g(v: np.ndarray) -> list:
    """CPython's "%g", or "" where it needs the exponent form (the device writer hands those values back)."""
    return [s if "e" not in s else "" for s in ("%g" % x for x in v.astype(np.float64).tolist())]


def device_g(ctx, v: np.ndarray) -> list:
    out = ctx.test_format_g(v)
    n = out[:, 15].astype(np.int64)
    assert (n <= 15).all()
    keep = np.arange(16)[None, :] < n[:, None]
    assert not out[:, :15][~keep[:, :15]].any(), "bytes after the text are not zero"
    slots = out.copy()
    slots[np.arange(len(n)), n] = ord("\n")
    return slots[np.arange(16)[None, :] <= n[:, None]].tobytes().decode().split("\n")[:-1]


def assert_format_g(ctx, v: np.ndarray, what: str):
    got, want = device_g(ctx, v), expected_g(v)
    assert len(got) == len(want) == v.size
    if got != want:
        bad = [i for i in range(v.size) if got[i] != want[i]]
        show = ", ".join(f"{float(v[i])!r}: device {got[i]!r}, %g {want[i]!r}" for i in bad[:8])
        pytest.fail(f"{what}: {len(bad)} of {v.size} values differ from %g ({show})")


def test_format_g_every_tie_and_its_neighbours(gpu_ctx):
    t = ties()
    # per decade X = -4 .. 5: 1, 3, 12, 58, 288, 1440, 7200, 36000, 180000, 900000
    assert t.size == 1_125_002
    assert_format_g(gpu_ctx, _ulp_neighbours(t), "ties")


def test_format_g_decade_boundaries_and_seventh_digit_carries(gpu_ctx):
    win = [_window(F32(10.0 ** j), 1 << 14) for j in range(-4, 7)]
    # 9.999995 -> "10", 99999.95 -> "100000", 999999.5 -> exponent form: the rounding carries into a seventh digit
    win += [_window(F32(10.0 ** j * (1 - 5e-7)), 1 << 14) for j in range(-3, 7)]
    assert_format_g(gpu_ctx, np.concatenate(win), "powers of ten and carries")


def test_format_g_random_bit_patterns_and_one_binade(gpu_ctx):
    rng = np.random.default_rng(2024)
    r = rng.integers(_bits(1e-4), _bits(1e6), size=1_000_000, dtype=np.uint32).view(F32)
    assert_format_g(gpu_ctx, r, "random bit patterns")
    assert_format_g(gpu_ctx, np.arange(_bits(64.0), _bits(128.0), dtype=np.uint32).view(F32), "[64, 128)")


def test_format_g_values_handed_back(gpu_ctx):
    edges = np.array([np.float32(1e-45), np.finfo(F32).tiny, F32(9.9999e-5), F32(1e6),
                      np.nextafter(F32(1e6), F32(np.inf)), np.finfo(F32).max, np.inf, -np.inf, np.nan, -1.5, -1e-4,
                      -np.finfo(F32).max, F32(3e-5), F32(2.5e7)], F32)
    out = gpu_ctx.test_format_g(np.concatenate([np.zeros(1, F32), edges]))
    assert out[0, 15] == 1 and bytes(out[0, :1]) == b"0"
    assert (out[1:, 15] == 0).all(), [float(x) for x in edges[out[1:, 15] != 0]]
    # %g decides on the value rounded to six digits: just under 1e-4 is still 0.0001, just under 1e6 is 1e+06
    near = np.array([F32(1e-4), np.nextafter(F32(1e-4), F32(0)), np.nextafter(F32(1e6), F32(0))], F32)
    assert device_g(gpu_ctx, near) == ["0.0001", "0.0001", ""] == expected_g(near)


# ---------------------------------------------------------------------------------------------------------------
# BGZF encoder
# ---------------------------------------------------------------------------------------------------------------
HOST_MODEL = {0: "ugvc_test_deflate_block_lanes", 1: "ugvc_test_deflate_block"}  # encoder -> its host restatement


def host_block(L, encoder: int, data: bytes) -> bytes:
    src = np.frombuffer(data + b"\0" * 8, dtype=np.uint8).copy()
    out = np.zeros(65536, dtype=np.uint8)
    n = getattr(L, HOST_MODEL[encoder])(src.ctypes.data_as(C.c_void_p), len(data), out.ctypes.data_as(C.c_void_p))
    assert n > 0, n
    return out[:n].tobytes()


def check_device_deflate(ctx, L, data: bytes, encoder: int, name: str) -> list:
    comp, csize = ctx.test_device_deflate(data, encoder)
    n_blocks = (len(data) + CHUNK - 1) // CHUNK
    assert len(csize) == n_blocks and int(csize.sum()) == len(comp), name
    blocks, at = [], 0
    for b in range(n_blocks):
        part = data[b * CHUNK:(b + 1) * CHUNK]
        blk = comp[at:at + int(csize[b])]
        assert blk[:16] == b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0", (name, b)
        assert struct.unpack_from("<H", blk, 16)[0] + 1 == len(blk) <= 65536, (name, b)
        assert zlib.decompress(blk[18:-8], -15) == part, (name, b)
        assert struct.unpack_from("<II", blk, len(blk) - 8) == (zlib.crc32(part) & 0xFFFFFFFF, len(part)), (name, b)
        assert blk == host_block(L, encoder, part), f"{name}: block {b} differs from {HOST_MODEL[encoder]}"
        blocks.append(blk)
        at += len(blk)
    assert b"".join(blocks) == comp  # packed back to back at the scanned offsets
    if n_blocks:
        assert gzip.decompress(comp) == data, name
    assert ctx.test_device_deflate(data, encoder)[0] == comp, f"{name}: a second run gives other bytes"
    return blocks


def _rnd(rng, n, lo=0, hi=256) -> bytes:
    return rng.integers(lo, hi, size=n, dtype=np.uint8).tobytes()


def _repeat(unit: bytes, n: int) -> bytes:
    return (unit * (n // len(unit) + 1))[:n]


def _far_repeat(rng, period: int, copies: int) -> bytes:
    """A chunk of `period` bytes repeated: 256 random bytes then zeros, so that the random part's 4-byte prefixes
    stay in the encoder's hash table until the copy, exactly `period` bytes later."""
    unit = _rnd(rng, 256) + b"\0" * (period - 256)
    return unit * copies


def deflate_inputs(text: bytes) -> dict:
    rng = np.random.default_rng(23)
    cases = {}
    for n in (0, 1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 257, 258, 259, 260, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 17):
        cases[f"vcf[{n}]"] = _repeat(text, n) if n else b""
        cases[f"A[{n}]"] = b"A" * n
    cases["vcf text"] = text
    cases["random"] = _rnd(rng, 3 * CHUNK + 17)                      # the stored fallback
    cases["random 0x90..0xff"] = _rnd(rng, 2 * CHUNK + 5, 0x90)      # stored, every byte a 9-bit literal
    words = [_rnd(rng, int(rng.integers(3, 40)), 0x90) for _ in range(64)]
    cases["words of 0x90..0xff"] = b"".join(words[int(k)] for k in rng.integers(0, 64, size=9000))  # 9-bit literals, compressed
    cases["zeros"] = b"\0" * (2 * CHUNK + 5)
    cases["all A"] = b"A" * (2 * CHUNK + 5)
    for p in (2, 3, 31, 32, 33):
        cases[f"period {p}"] = _repeat(_rnd(rng, p), CHUNK + 1000)
    cases["repeat 32768"] = _far_repeat(rng, 32768, 4)   # matches at exactly the largest distance DEFLATE allows
    cases["repeat 32769"] = _far_repeat(rng, 32769, 4)   # ... and one beyond it: must not be matched
    runs = []
    for _ in range(40):
        for r in (258, 259, 260):
            runs += [_rnd(rng, int(rng.integers(1, 40))), bytes([int(rng.integers(0, 256))]) * r]
    cases["runs 258..260"] = b"".join(runs)
    return cases


def mixed_input(cases: dict, n_blocks: int = 40) -> bytes:
    """Pieces of every other input, of random lengths, until n_blocks blocks (the last one short)."""
    rng = np.random.default_rng(41)
    srcs = [v for v in cases.values() if len(v) > 1000]
    parts, total, want = [], 0, (n_blocks - 1) * CHUNK + 12345
    while total < want:
        s = srcs[int(rng.integers(0, len(srcs)))]
        a = int(rng.integers(0, len(s) - 1))
        piece = s[a:a + int(rng.integers(100, 30000))]
        parts.append(piece)
        total += len(piece)
    return b"".join(parts)[:want]


@pytest.fixture(scope="module")
def job():
    ds = util.make_dataset(n_records=2000, n_custom=4, seed=57)
    _, tr, x = util.fit_transformer(ds)
    model = util.fit_model("gb_small", x, ds["labels"])
    plan = MC.compile_plan(VcfHeader(ds["header_text"]), tr, model, ds["customs"])
    return ds, plan


@pytest.fixture()
def enc_ctx(gpu_ctx, job):
    gpu_ctx.load_plan(job[1].blob)
    gpu_ctx.reserve(48 * CHUNK, 4096, 1)  # the writer's buffer holds the 40-block input
    return gpu_ctx


@pytest.mark.parametrize("encoder", [0, 1], ids=["warp", "thread"])
def test_device_deflate_edges(enc_ctx, job, encoder):
    L = lib.load_library()
    cases = deflate_inputs(job[0]["text"])
    cases["mix of 40 blocks"] = mixed_input(cases)
    for name, data in cases.items():
        check_device_deflate(enc_ctx, L, data, encoder, name)
    assert (len(cases["mix of 40 blocks"]) + CHUNK - 1) // CHUNK == 40


@pytest.mark.parametrize("encoder", [0, 1], ids=["warp", "thread"])
def test_device_deflate_uses_distance_32768(enc_ctx, encoder):
    """The repeated chunk of 32768 bytes is found exactly one period back: its random part costs a match, not 256
    literals.  (One byte more and the same chunk is out of reach: its literals come back.)"""
    L = lib.load_library()
    rng = np.random.default_rng(7)
    sizes = {}
    for period in (32768, 32769):
        rep = _far_repeat(rng, period, 2)[:CHUNK]
        other = rep[:period] + _far_repeat(rng, period, 1)[:CHUNK - period]  # same shape, a fresh random part
        sizes[period] = [len(check_device_deflate(enc_ctx, L, d, encoder, f"{period}")[0]) for d in (rep, other)]
    assert sizes[32768][0] + 150 < sizes[32768][1], sizes
    assert abs(sizes[32769][0] - sizes[32769][1]) < 16, sizes


# ---------------------------------------------------------------------------------------------------------------
# first record at or after a text offset
# ---------------------------------------------------------------------------------------------------------------
def test_first_records_is_a_lower_bound_on_the_line_starts(gpu_ctx, job):
    ds, plan = job
    gpu_ctx.load_plan(plan.blob)
    gpu_ctx.set_key_order(*lib.learn_key_order(ds["text"]))
    gpu_ctx.reserve(len(ds["text"]) + (1 << 20), len(ds["lines"]) + 64, 1)
    text = ds["text"]
    comp = np.frombuffer(bgzf_io.compress_bytes(text), dtype=np.uint8)
    got = gpu_ctx.filter_bgzf(comp, 0, len(text), 30.0, 0, len(ds["lines"]) + 64)
    assert got is not None and got["n_records"] == len(ds["lines"])
    nl = np.flatnonzero(np.frombuffer(text, dtype=np.uint8) == 10)
    starts = np.concatenate([[0], nl[:-1] + 1]).astype(np.int64)
    assert starts.size == got["n_records"]
    offsets = np.unique(np.concatenate([[0], starts, starts - 1, starts + 1, np.arange(0, len(text) + 1, 0xFF00),
                                        [len(text), len(text) + 1]]))
    offsets = offsets[offsets >= 0].astype(np.uint64)
    want = np.searchsorted(starts, offsets.astype(np.int64), "left")
    # the call takes as many offsets as the lane's scan scratch holds: 16 always fit
    res = np.concatenate([gpu_ctx.filter_bgzf_first_records(offsets[i:i + 16]) for i in range(0, offsets.size, 16)])
    bad = np.flatnonzero(res != want)
    assert bad.size == 0, [(int(offsets[i]), int(res[i]), int(want[i])) for i in bad[:8]]
    assert want[-1] == want[-2] == starts.size  # past the last line start: the record count


# ---------------------------------------------------------------------------------------------------------------
# the range and capacity refusals of the file-path entry points
# ---------------------------------------------------------------------------------------------------------------
WHO = {"filter_bgzf_edits": "filter_bgzf", "filter_bgzf_split": "filter_bgzf_split", "afr_bgzf": "afr_bgzf",
       "bsn_bgzf": "bsn_bgzf", "hcr_scan": "hcr_scan"}
# out_capacity too small: the filter calls hand the range to the host writer, the tools refuse the argument
OUT_TOO_SMALL = {"filter_bgzf_edits": lib.UGVC_E_FALLBACK, "filter_bgzf_split": lib.UGVC_E_FALLBACK,
                 "afr_bgzf": lib.UGVC_E_ARG, "bsn_bgzf": lib.UGVC_E_ARG}


def _call(entry: str, j: dict, comp: np.ndarray, skip_head: int, take_bytes: int, capacity_records: int,
          out_capacity: int) -> tuple[int, int, str]:
    """(rc, *out_n_records, ugvc_last_error) of one call of `entry` through ctypes, every output buffer sized for the
    whole range and the capacities as given."""
    ctx, n_max = j["ctx"], j["n_max"]
    out = np.empty(len(j["text"]) * 2 + (1 << 20), np.uint8)
    assert out_capacity <= out.size
    blocks = np.empty(out.size // 65536 + 8, np.uint32)
    ri, ls, ls2 = np.empty(n_max, lib.RECINFO_DTYPE), np.empty(n_max + 1, np.int64), np.empty(n_max + 1, np.int64)
    u8, i64, i32, runs = np.empty(n_max, np.uint8), np.empty(n_max, np.int64), np.empty(n_max, np.int32), np.empty((n_max, 2), np.int64)
    stats = np.zeros(8, np.int64)
    nb, nblk, n, x = C.c_size_t(), C.c_size_t(), C.c_int64(-1), C.c_int64()
    p = lib._ptr  # noqa: SLF001
    src = (p(comp), comp.size, skip_head, take_bytes)
    tail = (p(out), out_capacity, C.byref(nb), p(blocks), blocks.size, C.byref(nblk), p(ri), p(ls))
    if entry in ("filter_bgzf_edits", "filter_bgzf_split"):
        e, keep = lib._file_edits(True, False, j.get("blacklists"), None)  # noqa: F841, SLF001  (keep: alive for the call)
        if entry == "filter_bgzf_edits":
            rc = lib.load_library().ugvc_filter_bgzf_edits(ctx.h, 0, *src, 30.0, 0, C.byref(e), *tail, p(u8), capacity_records,
                                                           C.byref(n))
        else:
            ma = j["ma"]
            rc = lib.load_library().ugvc_filter_bgzf_split(ctx.h, j["index_ctx"].h, ma.h, 0, *src, p(ma.ref), ma.ref.size, 30.0,
                                                           0, C.byref(e), *tail, p(u8), capacity_records, C.byref(n), p(stats))
    elif entry == "afr_bgzf":
        rc = lib.load_low_af_ratio().ugvc_afr_bgzf(ctx.h, 0, *src, 0, C.byref(j["params"]), *tail, p(i64), p(u8),
                                                   capacity_records, C.byref(n), C.byref(x))
    elif entry == "bsn_bgzf":
        rc = lib.load_bridging_snvs().ugvc_bsn_bgzf(ctx.h, 0, *src, 0, C.byref(j["params"]), *tail, p(ls2), p(i64), p(u8), p(i32),
                                                    capacity_records, C.byref(n), C.byref(x))
    else:
        rc = lib.load_gvcf_hcr().ugvc_hcr_scan(ctx.h, 0, *src, C.byref(j["params"]), capacity_records, C.byref(n), p(stats),
                                               p(runs))
    return rc, n.value, lib.load_library().ugvc_last_error(ctx.h).decode()


@pytest.mark.parametrize("entry", list(WHO))
def test_range_and_capacity_refusals(gpu_ctx, job, request, entry):
    from tests.test_gpu_x_inflate_edges import ENTRIES

    j = ENTRIES[entry][0](gpu_ctx, job[0], request)
    text, who = j["text"], WHO[entry]
    comp = np.frombuffer(bgzf_io.compress_bytes(text), dtype=np.uint8)
    n_lines, big = text.count(b"\n"), len(text) * 2 + (1 << 20)
    assert _call(entry, j, comp, 0, 0, j["n_max"], big)[:2] == (lib.UGVC_OK, n_lines)
    assert _call(entry, j, comp, len(text) + 1, 0, j["n_max"], big)[::2] == (
        lib.UGVC_E_ARG, f"{who}: skip_head beyond the inflated blocks")
    assert _call(entry, j, comp, 0, len(text) + 1, j["n_max"], big)[::2] == (
        lib.UGVC_E_ARG, f"{who}: the range is longer than the inflated blocks")
    assert _call(entry, j, comp, 0, 0, n_lines - 1, big) == (
        lib.UGVC_E_ARG, n_lines, f"{who}: output capacity smaller than the record count")
    if entry in OUT_TOO_SMALL:
        assert _call(entry, j, comp, 0, 0, j["n_max"], 16)[::2] == (
            OUT_TOO_SMALL[entry], f"{who}: out_capacity smaller than the compressed output")
    assert _call(entry, j, comp, 0, 0, j["n_max"], big)[:2] == (lib.UGVC_OK, n_lines)  # nothing sticks to the lane
