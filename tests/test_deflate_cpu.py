"""CPU: the device BGZF encoder (csrc/deflate.cuh, compiled for the host) writes blocks that zlib inflates back to
the input, with the right CRC32 / ISIZE footer -- VCF text, runs, random bytes (stored fallback), edge sizes."""
import ctypes as C
import gzip
import struct
import zlib

import numpy as np

from tests import util
from variantcalling_b200 import lib

CHUNK = 57344


import pytest


@pytest.fixture(params=["ugvc_test_deflate_block", "ugvc_test_deflate_block_lanes"], autouse=True)
def encoder(request):
    """Both encoders: one thread per block (deflate.cuh: def_block) and the host model of the warp-per-block kernel."""
    global ENCODER
    ENCODER = request.param
    return request.param


ENCODER = "ugvc_test_deflate_block"


def encode(L, data: bytes) -> bytes:
    src = np.frombuffer(data + b"\0" * 8, dtype=np.uint8).copy()
    out = np.zeros(65536, dtype=np.uint8)
    n = getattr(L, ENCODER)(src.ctypes.data_as(C.c_void_p), len(data), out.ctypes.data_as(C.c_void_p))
    assert n > 0, n
    return out[:n].tobytes()


def check_block(block: bytes, data: bytes):
    assert block[:4] == b"\x1f\x8b\x08\x04" and block[12:14] == b"BC"
    bsize = struct.unpack_from("<H", block, 16)[0] + 1
    assert bsize == len(block) <= 65536
    crc, isize = struct.unpack_from("<II", block, len(block) - 8)
    assert isize == len(data) and crc == (zlib.crc32(data) & 0xFFFFFFFF)
    assert zlib.decompress(block[18:-8], -15) == data   # raw DEFLATE payload
    assert gzip.decompress(block) == data               # and as the gzip member it is


def test_vcf_text_round_trip_and_ratio():
    L = lib.load_library()
    ds = util.make_dataset(n_records=1200, n_custom=20, seed=3)
    text = ds["text"]
    total_in = total_out = 0
    for i in range(0, len(text), CHUNK):
        part = text[i:i + CHUNK]
        blk = encode(L, part)
        check_block(blk, part)
        total_in += len(part)
        total_out += len(blk)
    print(ENCODER, "ratio", total_in / total_out)
    assert total_out < 0.6 * total_in, (total_in, total_out)  # greedy LZ + fixed codes still shrinks VCF text well


def test_edge_inputs():
    L = lib.load_library()
    rng = np.random.default_rng(5)
    cases = [b"", b"A", b"AB", b"ABC", b"ABCD", b"ABCDABCD", b"A" * 300, b"A" * CHUNK, bytes(range(256)) * 200,
             rng.integers(0, 256, size=CHUNK, dtype=np.uint8).tobytes(),       # incompressible: stored
             rng.integers(0, 256, size=1000, dtype=np.uint8).tobytes(),
             (b"chr1\t12345\t.\tA\tG\t50\tPASS\tAC=1;AF=0.5\n" * 2000)[:CHUNK],
             b"\xff" * 70 + b"\x00" * 70 + b"\xff" * 700]
    # short periods: matches overlap their own source, one match covers whole 32-position windows
    for p in (2, 3, 31, 32, 33):
        cases.append((rng.integers(0, 256, size=p, dtype=np.uint8).tobytes() * (CHUNK // p + 1))[:CHUNK])
    # a chunk repeated exactly 32768 bytes later (the largest distance DEFLATE allows) and 32769 bytes later (beyond)
    for period in (32768, 32769):
        unit = rng.integers(0, 256, size=256, dtype=np.uint8).tobytes() + b"\0" * (period - 256)
        cases.append((unit * 2)[:CHUNK])
    # bytes >= 0x90 take 9-bit literal codes: stored when random, compressed when drawn from a vocabulary
    cases.append(rng.integers(0x90, 0x100, size=CHUNK, dtype=np.uint8).tobytes())
    words = [rng.integers(0x90, 0x100, size=int(rng.integers(3, 40)), dtype=np.uint8).tobytes() for _ in range(64)]
    cases.append(b"".join(words[int(k)] for k in rng.integers(0, 64, size=3000))[:CHUNK])
    # runs around the longest match (258) between random bytes
    for r in (257, 258, 259, 260):
        cases.append(b"".join(rng.integers(0, 256, size=20, dtype=np.uint8).tobytes() + b"R" * r for _ in range(50)))
    for data in cases:
        check_block(encode(L, data), data)


def test_random_structured_inputs():
    L = lib.load_library()
    rng = np.random.default_rng(11)
    words = [bytes(rng.integers(32, 127, size=int(rng.integers(1, 30)), dtype=np.uint8)) for _ in range(200)]
    for _ in range(30):
        n = int(rng.integers(1, CHUNK))
        data = b"".join(words[int(k)] for k in rng.integers(0, len(words), size=n // 8 + 1))[:n]
        check_block(encode(L, data), data)
