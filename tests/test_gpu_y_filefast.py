"""GPU: the device-side file path (ugvc_filter_bgzf: BGZF inflate -> K1..K3 -> record writer -> BGZF deflate) writes
exactly the text the host writer (ugvc_splice_records) produces from the host-buffer path's results, as valid BGZF
blocks, with line offsets that point at the records; ranges that start inside a block; the fallback signal."""
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


@pytest.fixture(scope="module")
def job():
    ds = util.make_dataset(n_records=6000, n_custom=6, seed=91)
    _, tr, x = util.fit_transformer(ds)
    model = util.fit_model("gb_small", x, ds["labels"])
    plan = MC.compile_plan(VcfHeader(ds["header_text"]), tr, model, ds["customs"])
    return ds, plan


# every FILTER column the writer's rule has to get right (pieces split on ';', empty ones dropped, PASS dropped when
# the record fails, LOW_SCORE added once)
FILTERS = [".", "PASS", "LOW_SCORE", "PASS;LOW_SCORE", "q10;PASS", "q10;;PASS", ";", "LOW_SCORE;LOW_SCORE", "PASSX"]


def crafted_lines(lines: list) -> list:
    """The records of `lines` with every FILTER of FILTERS, and in turn: a long QUAL, and alleles GGC / CCG
    (CG_NON_HMER_INDEL under FILE_BLACKLIST_CG).  Records without a sample or with QUAL "." are not here: the model's
    features need both, and the reference raises on them before anything is written."""
    out = []
    for i, line in enumerate(lines):
        c = line.split("\t")
        c[6] = FILTERS[i % len(FILTERS)]
        kind = (i // len(FILTERS)) % 4
        if kind == 1:
            c[5] = c[5] + "0" * 40 + "1"
        elif kind == 2:
            c[3], c[4] = "GGC", "G"
        elif kind == 3:
            c[3], c[4] = "C", "CCG"
        out.append("\t".join(c))
    return out


def host_text(ctx, text: bytes, flags: int, threshold: float = 30.0) -> bytes:
    """The host-buffer path + the host writer on the same records."""
    L = lib.load_library()
    res = ctx.filter_batch(text, threshold)
    n = res["n_records"]
    buf = np.frombuffer(text, dtype=np.uint8)
    out = np.empty(buf.size + n * 128 + 1024, dtype=np.uint8)
    out_ls = np.empty(n + 1, dtype=np.int64)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    code = table = off = None
    if flags & lib.FILE_BLACKLIST_CG:
        code = (res["recinfo"]["flags"] & 1).astype(np.int32)
        strings = [b"PASS", b"CG_NON_HMER_INDEL"]
        table = np.frombuffer(b"".join(strings), dtype=np.uint8)
        off = np.array([0, 4, 4 + len(strings[1])], dtype=np.int64)
    nb = L.ugvc_splice_records(p(buf), p(res["line_start"]), p(res["recinfo"]), p(res["low_score"]), p(res["qual"]), n,
                               int(bool(flags & lib.FILE_OVERWRITE_QUAL)), 1, p(code), p(table), p(off), None, 0, p(out),
                               out.size, p(out_ls), 4)
    assert nb > 0
    return out[:nb].tobytes(), res


def check_blocks(comp: bytes, csizes) -> bytes:
    at, parts = 0, []
    for cs in csizes:
        blk = comp[at:at + int(cs)]
        assert blk[:4] == b"\x1f\x8b\x08\x04" and struct.unpack_from("<H", blk, 16)[0] + 1 == len(blk)
        data = zlib.decompress(blk[18:-8], -15)
        crc, isize = struct.unpack_from("<II", blk, len(blk) - 8)
        assert isize == len(data) and crc == (zlib.crc32(data) & 0xFFFFFFFF)
        parts.append(data)
        at += int(cs)
    assert at == len(comp)
    return b"".join(parts)


FLAGS = [0, lib.FILE_BLACKLIST_CG, lib.FILE_OVERWRITE_QUAL | lib.FILE_BLACKLIST_CG]


@pytest.mark.parametrize(("data", "flags"), [("synthetic", f) for f in FLAGS] + [("crafted", f) for f in FLAGS],
                         ids=[str(f) for f in FLAGS] + [f"crafted-{f}" for f in FLAGS])
def test_device_file_path_equals_host_writer(gpu_ctx, job, data, flags):
    """The synthetic records as they are (threshold 30), and the crafted ones (crafted_lines) with the threshold at
    their median qual, so that half the records fail and every FILTER of FILTERS goes through both branches."""
    ds, plan = job
    gpu_ctx.load_plan(plan.blob)
    gpu_ctx.set_key_order(*lib.learn_key_order(ds["text"]))
    gpu_ctx.reserve(len(ds["text"]) + (1 << 20), len(ds["lines"]) + 64, 1)
    ds, threshold = dict(ds), 30.0
    if data == "crafted":
        ds["lines"] = crafted_lines(ds["lines"])
        ds["text"] = ("\n".join(ds["lines"]) + "\n").encode()
        threshold = float(np.median(gpu_ctx.filter_batch(ds["text"], 30.0)["qual"]))
    want, res = host_text(gpu_ctx, ds["text"], flags, threshold)
    if data == "crafted":
        low = res["low_score"].astype(bool)
        assert 0.4 < low.mean() < 0.6 and (res["recinfo"]["flags"] & 1).sum() > 1000
        for k, filt in enumerate(FILTERS):  # each FILTER on passing and on failing records
            assert low[k::len(FILTERS)].any() and not low[k::len(FILTERS)].all(), filt
    comp = np.frombuffer(bgzf_io.compress_bytes(ds["text"]), dtype=np.uint8)
    got = gpu_ctx.filter_bgzf(comp, 0, len(ds["text"]), threshold, flags, len(ds["lines"]) + 64)
    assert got is not None and got["n_records"] == res["n_records"]
    out = check_blocks(got["bgzf"].tobytes(), got["block_csize"])
    assert out == want, "the device writer's text differs from the host writer's"
    assert gzip.decompress(got["bgzf"].tobytes()) == want  # a plain gzip reader agrees
    ls = got["line_start"]
    lines = want.split(b"\n")
    for i in (0, 1, len(lines) // 2, res["n_records"] - 1):
        assert want[ls[i]:ls[i + 1] - 1] == lines[i]
    assert np.array_equal(got["low_score"], res["low_score"])
    assert all(int(c) <= 65536 for c in got["block_csize"]) and len(got["block_csize"]) == (len(want) + lib.DEF_CHUNK - 1) // lib.DEF_CHUNK


def test_range_inside_blocks(gpu_ctx, job):
    """A contig of an indexed file starts and ends inside BGZF blocks: skip_head / take_bytes select the lines."""
    ds, plan = job
    gpu_ctx.load_plan(plan.blob)
    gpu_ctx.set_key_order(*lib.learn_key_order(ds["text"]))
    gpu_ctx.reserve(len(ds["text"]) + (1 << 20), len(ds["lines"]) + 64, 1)
    lines = ds["lines"]
    a, b = 1500, 4200
    head = ("\n".join(lines[:a]) + "\n").encode()
    mid = ("\n".join(lines[a:b]) + "\n").encode()
    comp = bgzf_io.compress_bytes(ds["text"])
    # blocks hold 0xff00 bytes each: the range starts in block len(head) // 0xff00
    blk = 0xff00
    first = len(head) // blk
    sizes, at = [], 0
    while at < len(comp):
        sizes.append(struct.unpack_from("<H", comp, at + 16)[0] + 1)
        at += sizes[-1]
    c0 = sum(sizes[:first])
    part = np.frombuffer(comp[c0:], dtype=np.uint8)
    want, _ = host_text(gpu_ctx, mid, 0)
    got = gpu_ctx.filter_bgzf(part, len(head) - first * blk, len(mid), 30.0, 0, len(lines) + 64)
    assert got is not None and got["n_records"] == b - a
    assert gzip.decompress(got["bgzf"].tobytes()) == want


def test_fallback_when_the_general_writer_is_needed(gpu_ctx, job):
    ds, plan = job
    gpu_ctx.load_plan(plan.blob)
    gpu_ctx.set_key_order(*lib.learn_key_order(ds["text"]))
    gpu_ctx.reserve(len(ds["text"]) + (1 << 20), len(ds["lines"]) + 64, 1)
    lines = list(ds["lines"][:400])
    cols = lines[7].split("\t")
    cols[7] = cols[7] + ";TREE_SCORE=12.5"  # already filtered once: the key has to be replaced, not appended
    lines[7] = "\t".join(cols)
    text = ("\n".join(lines) + "\n").encode()
    comp = np.frombuffer(bgzf_io.compress_bytes(text), dtype=np.uint8)
    assert gpu_ctx.filter_bgzf(comp, 0, len(text), 30.0, 0, 512) is None
    # the same records without that line go through
    del lines[7]
    text = ("\n".join(lines) + "\n").encode()
    comp = np.frombuffer(bgzf_io.compress_bytes(text), dtype=np.uint8)
    got = gpu_ctx.filter_bgzf(comp, 0, len(text), 30.0, 0, 512)
    assert got is not None and gzip.decompress(got["bgzf"].tobytes()) == host_text(gpu_ctx, text, 0)[0]


def _with_info(new_info):
    def edit(line: str) -> str:
        c = line.split("\t")
        c[7] = new_info(c[7])
        return "\t".join(c)
    return edit


# lines the device writer hands back to the host writer (UGVC_E_FALLBACK), and why
HANDED_BACK = {
    "TREE_SCORE": _with_info(lambda info: info + ";TREE_SCORE=12.5"),      # the key is replaced, not appended
    "BLACKLST": _with_info(lambda info: "BLACKLST=CG_NON_HMER_INDEL;" + info),
    "XTREE_SCORE": _with_info(lambda info: info + ";XTREE_SCORE=3"),       # the device matches the keys conservatively
    "XBLACKLST": _with_info(lambda info: info.replace(";", ";XBLACKLST=1;", 1)),
    "empty piece": _with_info(lambda info: info.replace(";", ";;", 1)),
    "leading ;": _with_info(lambda info: ";" + info),
    "trailing ;": _with_info(lambda info: info + ";"),
    "long line": _with_info(lambda info: info + ";NOTE=" + "x" * 70000),  # offsets past 65535 saturate in recinfo
}


@pytest.mark.parametrize("case", list(HANDED_BACK))
def test_lines_the_device_writer_hands_back(gpu_ctx, job, case):
    """One such line makes the call hand back; the same records without it go through and equal the host writer (a
    hand-back on clean records would be a silent slowdown: the tool takes the host path without a word)."""
    ds, plan = job
    gpu_ctx.load_plan(plan.blob)
    gpu_ctx.set_key_order(*lib.learn_key_order(ds["text"]))
    gpu_ctx.reserve(len(ds["text"]) + (1 << 20), len(ds["lines"]) + 64, 1)
    lines = list(ds["lines"][:300])
    for at in (0, 150, 299):
        edited = lines[:at] + [HANDED_BACK[case](lines[at])] + lines[at + 1:]
        text = ("\n".join(edited) + "\n").encode()
        assert gpu_ctx.filter_batch(text, 30.0)["n_records"] == len(edited)  # the records themselves are fine
        comp = np.frombuffer(bgzf_io.compress_bytes(text), dtype=np.uint8)
        for flags in FLAGS:
            assert gpu_ctx.filter_bgzf(comp, 0, len(text), 30.0, flags, 512) is None, (case, at, flags)
        clean = ("\n".join(lines[:at] + lines[at + 1:]) + "\n").encode()
        comp = np.frombuffer(bgzf_io.compress_bytes(clean), dtype=np.uint8)
        for flags in FLAGS:
            got = gpu_ctx.filter_bgzf(comp, 0, len(clean), 30.0, flags, 512)
            assert got is not None, f"clean records handed back ({case}, {at}, {flags})"
            assert gzip.decompress(got["bgzf"].tobytes()) == host_text(gpu_ctx, clean, flags)[0]
