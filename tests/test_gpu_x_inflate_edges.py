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


def _split_vcf(full: str) -> tuple[str, bytes]:
    """(header, data lines) of a whole VCF text."""
    at = full.index("\n", full.index("#CHROM")) + 1
    return full[:at], full[at:].encode()


def _reserved(ctx, plan_blob: bytes, text: bytes, phreds: int = 0, grow: int = 1):
    """The plan loaded and one lane reserved for `text`, or for `grow` times its bytes and lines (a split's scored pass)."""
    ctx.load_plan(plan_blob)
    if phreds:
        ctx.enable_phreds(phreds)
    ctx.reserve(grow * len(text) + (1 << 20), grow * text.count(b"\n") + 64, 1)


def _bound(load):
    """Bind a tool's entry points, or skip where the library lacks them (the host emulation of the filter path)."""
    try:
        load()
    except AttributeError:
        pytest.skip("the library lacks the tool's entry points: not part of the host emulation")


# The device file-path entry points on one context each: set-up(gpu_ctx, ds, request) -> a job dict with the input
# "text", the context "ctx", "n_max" (records the outputs hold) and what the entry needs besides.  run(job, bgzf bytes) ->
# (record count, output bytes), or None where the entry hands the range back (the host emulation's stubs).
def _setup_filter(ctx, ds, _request):
    _, tr, x = util.fit_transformer(ds)
    plan = MC.compile_plan(VcfHeader(ds["header_text"]), tr, util.fit_model("lr", x, ds["labels"]), ds["customs"])
    _reserved(ctx, plan.blob, ds["text"])
    pos = np.unique([int(ln.split("\t", 2)[1]) for ln in ds["lines"][::7]]).astype(np.int64)
    return {"text": ds["text"], "ctx": ctx, "n_max": len(ds["lines"]) + 64, "blacklists": [("BL_A;PASS", pos)]}


def _setup_split(_ctx, _ds, request):
    from tests.test_multiallelics_cpu import contig_text
    from variantcalling_b200 import multiallelics as PM

    mds, tr, model, _ = util.make_multiallelic_case(12, "lr")
    hdr = VcfHeader(mds["header_text"])
    text = contig_text(mds, "chrM1")
    ctx, index_ctx = lib.Context(0), lib.Context(0)
    ma = PM.DeviceSplitPlan(hdr, hdr.loader_columns(mds["customs"]), mds["ref"]["chrM1"])
    for closer in (ctx.close, index_ctx.close, ma.close):
        request.addfinalizer(closer)
    _reserved(ctx, MC.compile_plan(hdr, tr, model, mds["customs"]).blob, text, phreds=2, grow=4)
    _reserved(index_ctx, MC.compile_plan_no_model(hdr).blob, text)
    return {"text": text, "ctx": ctx, "index_ctx": index_ctx, "ma": ma, "n_max": text.count(b"\n") + 64}


def _setup_afr(ctx, _ds, _request):
    from tests import low_af_ratio_data as LD

    _bound(lib.load_low_af_ratio)
    head, text = _split_vcf(LD.random_text(4000, 2, 21))
    _reserved(ctx, MC.compile_plan_no_model(VcfHeader(head)).blob, text)
    params = LD.params(head, af_ratio_threshold=5, af_ratio_threshold_h_indels=2, t_vaf_threshold=0.2)
    return {"text": text, "ctx": ctx, "n_max": text.count(b"\n") + 64, "params": params}


def _setup_bsn(ctx, _ds, request):
    from tests import bridging_snvs_data as BD

    _bound(lib.load_bridging_snvs)
    g = BD.genome()
    head, text = _split_vcf(BD.text(BD.random_records(g, 4000, 31)))
    for name, seq in g.items():
        ctx.bsn_add_contig(name, seq)
    request.addfinalizer(ctx.bsn_clear_contigs)
    _reserved(ctx, MC.compile_plan_no_model(VcfHeader(head)).blob, text)
    return {"text": text, "ctx": ctx, "n_max": text.count(b"\n") + 64, "params": BD.params(head)}


def _setup_hcr(ctx, _ds, _request):
    from tests import gvcf_hcr_data as HD
    from variantcalling_b200 import gvcf_hcr

    _bound(lib.load_gvcf_hcr)
    head, text = _split_vcf(HD.text(HD.random_records(4000, 7)))
    _reserved(ctx, MC.compile_plan_no_model(VcfHeader(head)).blob, text)
    return {"text": text, "ctx": ctx, "n_max": text.count(b"\n") + 64, "params": gvcf_hcr.hcr_params(VcfHeader(head))}


def _run_filter(job, data):
    res = job["ctx"].filter_bgzf(np.frombuffer(data, np.uint8), 0, 0, 30.0, 0, job["n_max"])
    return None if res is None else (res["n_records"], res["bgzf"].tobytes())


def _run_edits(job, data):
    res = job["ctx"].filter_bgzf_edits(np.frombuffer(data, np.uint8), 0, 0, 30.0, 0, job["n_max"], blacklists=job["blacklists"])
    return None if res is None else (res["n_records"], res["bgzf"].tobytes(), res["n_blacklisted"])


def _run_split(job, data):
    res = job["ma"].filter_bgzf(job["ctx"], job["index_ctx"], np.frombuffer(data, np.uint8), 0, 0, 30.0, 0, job["n_max"])
    return None if res is None else (res["n_records"], res["bgzf"].tobytes())


def _run_afr(job, data):
    res = job["ctx"].afr_bgzf(np.frombuffer(data, np.uint8), 0, 0, False, job["params"], job["n_max"])
    return res["n_records"], res["bgzf"].tobytes()


def _run_bsn(job, data):
    res = job["ctx"].bsn_bgzf(np.frombuffer(data, np.uint8), 0, 0, False, job["params"], job["n_max"])
    return res["n_records"], res["bgzf"].tobytes()


def _run_hcr(job, data):
    ctx = job["ctx"]
    res = ctx.hcr_scan(np.frombuffer(data, np.uint8), 0, 0, job["params"], job["n_max"])
    return res["n_records"], ctx.hcr_emit(job["params"], False, -1, len(job["text"]) + 48 * res["n_records"] + 64)["bed"]


ENTRIES = {"filter_bgzf": (_setup_filter, _run_filter), "filter_bgzf_edits": (_setup_filter, _run_edits),
           "filter_bgzf_split": (_setup_split, _run_split), "afr_bgzf": (_setup_afr, _run_afr),
           "bsn_bgzf": (_setup_bsn, _run_bsn), "hcr_scan": (_setup_hcr, _run_hcr)}


def _refuses_and_names_the_first_bad_block(gpu_ctx, ds, request, entry):
    setup, run = ENTRIES[entry]
    job = setup(gpu_ctx, ds, request)
    good, crc_bad, inc_bad, text = _bad_files(job["text"])
    try:
        res = run(job, good)
    except lib.UgvcError as e:
        if "host emulation" not in e.message:
            raise
        res = None
    if res is None:
        pytest.skip(f"the device file path of {entry} is not part of the host emulation")
    assert res[0] == text.count(b"\n")
    for bad, where in ((crc_bad, r"block 1, code 9\)"), (inc_bad, r"block 2, code 3\)")):
        with pytest.raises(lib.UgvcError, match=where) as e:
            run(job, bad)
        assert e.value.code == lib.UGVC_E_IO
    assert run(job, good) == res


def test_filter_bgzf_refuses_and_names_the_first_bad_block(gpu_ctx, ds, request):
    _refuses_and_names_the_first_bad_block(gpu_ctx, ds, request, "filter_bgzf")


@pytest.mark.parametrize("entry", [e for e in ENTRIES if e != "filter_bgzf"])
def test_file_path_entry_refuses_and_names_the_first_bad_block(gpu_ctx, ds, request, entry):
    """The other device file-path entry points refuse the same blocks, and take a good input afterwards."""
    _refuses_and_names_the_first_bad_block(gpu_ctx, ds, request, entry)


def test_isize_zero_blocks_are_skipped_as_the_host_reader_skips_them(ictx):
    a = b"x" * 100
    data = D.bgzf_block(_raw(a, 6), a) + D.bgzf_block(b"\xff\xff", isize=0, crc=1) + IC.BGZF_EOF
    got, rc = inflate(ictx, data, 1)
    assert rc.tolist() == [0] and got.tobytes() == a
