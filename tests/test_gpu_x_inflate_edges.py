"""GPU: both device BGZF decoders (csrc/inflate.cuh; 0 = one warp per block, the default, 1 = one thread per block)
against zlib and the host reader's rule on crafted streams (tests/inflate_cases.py) and on a mutated corpus.

Through the test hook ugvc_test_device_inflate, which runs the product's staging and kernels with the decoder named and
reports the INF_* code of every block.  The host emulation has the thread decoder only: the warp decoder's tests skip
there.  The host reader's rule (hostio.cpp: inflate_block, htslib's) is restated in deflate_craft.host_rule; the fuzz
also runs the corpus through ugvc_bgzf_inflate_file to confirm the restatement."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

from tests import deflate_craft as D
from tests import inflate_cases as IC
from tests import util
from variantcalling_b200 import bgzf_io, lib
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader

pytestmark = pytest.mark.gpu
DECODERS = [pytest.param(0, id="warp"), pytest.param(1, id="thread")]


@pytest.fixture(scope="module")
def ds():
    return util.make_dataset(n_records=3000, n_custom=3, seed=41)


@pytest.fixture()
def ictx(gpu_ctx, ds):
    gpu_ctx.load_plan(MC.compile_plan_no_model(VcfHeader(ds["header_text"])).blob)
    gpu_ctx.reserve(64 << 20, 4096, 1)
    return gpu_ctx


def inflate(ctx, data: bytes, decoder: int):
    try:
        return ctx.test_device_inflate(data, decoder)
    except lib.UgvcError as e:
        if e.code == lib.UGVC_E_STATE and decoder == 0 and "host emulation" in e.message:
            pytest.skip("the warp-per-block decoder is not part of the host emulation")
        raise


def expected(blocks) -> tuple[list[bytes | None], list[int]]:
    """The host rule's output for every block with ISIZE > 0 (None: refused), and their ISIZEs."""
    outs, sizes = [], []
    for b in blocks:
        for payload, crc, isize in D.split_bgzf(b):
            if isize:
                outs.append(D.host_rule(payload, isize, crc))
                sizes.append(isize)
    return outs, sizes


@pytest.mark.parametrize("decoder", DECODERS)
@pytest.mark.parametrize("case", sorted(IC.VALID))
def test_crafted_shapes_equal_zlib(ictx, decoder, case):
    blocks = IC.VALID[case]()
    want, _ = expected(blocks)
    assert all(w is not None for w in want)
    got, rc = inflate(ictx, b"".join(blocks), decoder)
    assert rc.tolist() == [0] * len(want)
    assert got.tobytes() == b"".join(want)


@pytest.mark.parametrize("decoder", DECODERS)
def test_single_fault_refusals_have_their_codes(ictx, decoder):
    cases = IC.refusal_cases()
    names = sorted(cases)
    # between good blocks, so that a decoder that leaks state from one block to the next shows it
    good = D.bgzf_block(zlib.compress(b"good block\n" * 50, 9)[2:-4], b"good block\n" * 50)
    data = b"".join(cases[n][0] + good for n in names)
    _, rc = inflate(ictx, data, decoder)
    got = dict(zip(names, rc.tolist()[0::2]))
    assert got == {n: cases[n][1] for n in names}
    assert rc.tolist()[1::2] == [0] * len(names)


# ---------------------------------------------------------------------------------------------------------------
# differential fuzz against the host reader's rule
# ---------------------------------------------------------------------------------------------------------------
def _raw(data: bytes, level: int, strategy: int = zlib.Z_DEFAULT_STRATEGY) -> bytes:
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    return c.compress(data) + c.flush()


def _mutants(rng: random.Random, payload: bytes, crc: int, isize: int, k: int):
    yield payload, crc, isize
    for _ in range(k):
        p, c, n = bytearray(payload), crc, isize
        kind = rng.randrange(7)
        if kind == 0 and p:                                            # a bit anywhere
            i = rng.randrange(len(p))
            p[i] ^= 1 << rng.randrange(8)
        elif kind == 1 and p:                                          # a bit in the first 40 bytes: the dynamic header
            i = rng.randrange(min(40, len(p)))
            p[i] ^= 1 << rng.randrange(8)
        elif kind == 2 and p:                                          # a byte overwritten
            p[rng.randrange(len(p))] = rng.randrange(256)
        elif kind == 3 and p:                                          # truncated
            del p[rng.randrange(len(p)):]
        elif kind == 4:                                                # ISIZE - 1 / + 1
            n = isize + rng.choice((-1, 1)) if isize < 65536 else isize - 1  # noqa: PLR2004
        elif kind == 5:                                                # a CRC bit
            c ^= 1 << rng.randrange(32)
        else:                                                          # two bits in the header
            for _ in range(2):
                i = rng.randrange(min(40, len(p))) if p else 0
                if p:
                    p[i] ^= 1 << rng.randrange(8)
        if kind in (0, 1, 2, 6) and rng.random() < 0.5:  # noqa: PLR2004
            # resealed: ISIZE and CRC of what zlib makes of the changed stream, so that the decoding itself is compared
            d = zlib.decompressobj(-15)
            try:
                out = d.decompress(bytes(p), 65537)
            except zlib.error:
                out = None
            if out and d.eof and len(out) <= 65536:  # noqa: PLR2004
                c, n = zlib.crc32(out) & 0xFFFFFFFF, len(out)
        if n > 0:
            yield bytes(p), c, n


@pytest.fixture(scope="module")
def corpus(ds):
    """(BGZF bytes, [(payload, crc, isize)]) of >= 8000 seeded blocks: every crafted kind, zlib's levels 1 / 6 / 9,
    Z_FIXED and Z_RLE on VCF text and binary data, each mutated."""
    rng = random.Random(20261017)
    base = [blk for blocks in IC.valid_cases().values() for b in blocks for blk in D.split_bgzf(b) if blk[2]]
    base += [D.split_bgzf(b)[0] for b, _, _ in IC.refusal_cases().values()]
    text, noise = ds["text"], random.Random(7).randbytes(1 << 16)
    for src in (text, noise, bytes(range(256)) * 100):
        for size in (17, 300, 1500, 4000, 20000):
            at = rng.randrange(len(src) - size)
            piece = src[at:at + size]
            for level, strategy in ((1, 0), (6, 0), (9, 0), (6, zlib.Z_FIXED), (6, zlib.Z_RLE)):
                base.append((_raw(piece, level, strategy), zlib.crc32(piece) & 0xFFFFFFFF, size))
    blocks = []
    for payload, crc, isize in base:
        blocks += _mutants(rng, payload, crc, isize, 80 if isize <= 4096 else 6)  # noqa: PLR2004
    assert len(blocks) >= 8000, len(blocks)  # noqa: PLR2004
    data = b"".join(D.bgzf_block(p, isize=n, crc=c) for p, c, n in blocks)
    return data, blocks


@pytest.mark.parametrize("decoder", DECODERS)
def test_differential_fuzz_against_the_host_rule(ictx, corpus, decoder):
    data, blocks = corpus
    want = [D.host_rule(p, n, c) for p, c, n in blocks]
    got, rc = inflate(ictx, data, decoder)                             # every block in one call
    assert rc.size == len(blocks)
    off = np.concatenate([[0], np.cumsum([n for _, _, n in blocks])])
    accepted = [w is not None for w in want]
    assert min(sum(accepted), len(accepted) - sum(accepted)) >= 1000   # noqa: PLR2004  (both sides are exercised)
    bad = [(i, int(rc[i]), accepted[i]) for i in range(len(blocks)) if (rc[i] == 0) != accepted[i]]
    assert not bad, f"{len(bad)} blocks judged otherwise than the host rule, e.g. (index, code, rule accepts): {bad[:8]}"
    wrong = [i for i in range(len(blocks)) if accepted[i] and got[off[i]:off[i + 1]].tobytes() != want[i]]
    assert not wrong, wrong[:8]


def test_the_host_rule_is_the_host_readers(corpus, tmp_path):
    """ugvc_bgzf_inflate_file block by block over the same corpus: it accepts exactly what deflate_craft.host_rule
    accepts, with the same bytes."""
    data, blocks = corpus
    path = str(tmp_path / "corpus.gz")
    with open(path, "wb") as fh:
        fh.write(data)
    cl = lib.load_library()
    out = np.empty(65536, np.uint8)
    n = C.c_size_t()
    at, mismatched = 0, []
    for i, (p, c, isize) in enumerate(blocks):
        nxt = at + 26 + len(p)
        rc = cl.ugvc_bgzf_inflate_file(path.encode(), at << 16, nxt << 16 if nxt < len(data) else 0,
                                       out.ctypes.data_as(C.c_void_p), out.size, C.byref(n), 1)
        want = D.host_rule(p, isize, c)
        if (rc == 0) != (want is not None) or (rc == 0 and out[:n.value].tobytes() != want):
            mismatched.append((i, rc))
        at = nxt
    assert not mismatched, mismatched[:8]


# ---------------------------------------------------------------------------------------------------------------
# the product entry points
# ---------------------------------------------------------------------------------------------------------------
def _bad_files(text: bytes):
    """Six-block BGZF files of the whole lines of text's first 360 KB: intact, with the CRCs flipped in blocks 1 and 4,
    or with an incomplete code in blocks 2 and 5; and those lines."""
    text = text[:text.rfind(b"\n", 0, 360_000) + 1]
    cut = [i + 1 for i in range(len(text)) if text[i] == 10]
    cuts = [0] + [cut[len(cut) * k // 6 - 1] for k in range(1, 6)] + [len(text)]
    pieces = [text[cuts[k]:cuts[k + 1]] for k in range(6)]
    good = [D.bgzf_block(_raw(p, 6), p) for p in pieces]
    crc_bad = list(good)
    for k in (1, 4):
        crc_bad[k] = D.bgzf_block(_raw(pieces[k], 6), pieces[k], crc=zlib.crc32(pieces[k]) ^ 0x100)
    inc_bad = list(good)
    inc_block = IC.refusal_cases()["cl_incomplete"][0]
    for k in (2, 5):
        inc_bad[k] = inc_block
    return b"".join(good), b"".join(crc_bad), b"".join(inc_bad), text


def test_inflate_device_refuses_and_names_the_first_bad_block(ictx, ds):
    good, crc_bad, inc_bad, text = _bad_files(ds["text"])
    assert ictx.inflate_bgzf(good + bgzf_io.BGZF_EOF).tobytes() == text
    with pytest.raises(lib.UgvcError, match=r"block 1, code 9\)") as e:
        ictx.inflate_bgzf(crc_bad)
    assert e.value.code == lib.UGVC_E_IO
    with pytest.raises(lib.UgvcError, match=r"block 2, code 3\)") as e:
        ictx.inflate_bgzf(inc_bad)
    assert e.value.code == lib.UGVC_E_IO
    assert ictx.inflate_bgzf(good).tobytes() == text                   # nothing sticks to the context


def test_filter_bgzf_refuses_and_names_the_first_bad_block(gpu_ctx, ds):
    _, tr, x = util.fit_transformer(ds)
    plan = MC.compile_plan(VcfHeader(ds["header_text"]), tr, util.fit_model("lr", x, ds["labels"]), ds["customs"])
    gpu_ctx.load_plan(plan.blob)
    gpu_ctx.reserve(len(ds["text"]) + (1 << 20), len(ds["lines"]) + 64, 1)
    good, crc_bad, inc_bad, text = _bad_files(ds["text"])
    n_max = len(ds["lines"]) + 64
    res = gpu_ctx.filter_bgzf(np.frombuffer(good, np.uint8), 0, 0, 30.0, 0, n_max)
    if res is None:
        pytest.skip("the device record writer is not part of the host emulation")
    assert res["n_records"] == text.count(b"\n")
    for bad, where in ((crc_bad, r"block 1, code 9\)"), (inc_bad, r"block 2, code 3\)")):
        with pytest.raises(lib.UgvcError, match=where) as e:
            gpu_ctx.filter_bgzf(np.frombuffer(bad, np.uint8), 0, 0, 30.0, 0, n_max)
        assert e.value.code == lib.UGVC_E_IO
    again = gpu_ctx.filter_bgzf(np.frombuffer(good, np.uint8), 0, 0, 30.0, 0, n_max)
    assert again["bgzf"].tobytes() == res["bgzf"].tobytes()


def test_isize_zero_blocks_are_skipped_as_the_host_reader_skips_them(ictx):
    a = b"x" * 100
    data = D.bgzf_block(_raw(a, 6), a) + D.bgzf_block(b"\xff\xff", isize=0, crc=1) + IC.BGZF_EOF
    got, rc = inflate(ictx, data, 1)
    assert rc.tolist() == [0] and got.tobytes() == a
