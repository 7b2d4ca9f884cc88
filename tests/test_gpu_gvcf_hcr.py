"""GPU: gvcf_hcr on the device against oracle/gvcf_hcr_ref.py -- the BED text byte for byte and the skipped count of
gvcf_to_bed (gt True and False), the merged BED of gvcf_hcr and the CLI, the error contract, under pieces cut inside
overlap clusters and at contig changes, a record whose END covers the rest of its contig and records that overlap their
successor everywhere (no reset point), shorter and longer than the segment bound.
The test_hook_* tests run the kernels alone (ugvc_test_hcr) and also run on the host emulation
(tests/test_gvcf_hcr_emu_cpu.py)."""
import os

import numpy as np
import pytest

from oracle import gvcf_hcr_ref as R
from tests import gvcf_hcr_data as D
from variantcalling_b200 import bgzf_io, lib
from variantcalling_b200.vcf_header import VcfHeader

pytestmark = pytest.mark.gpu

REASONS = {"literal": lib.HCR_E_LITERAL, "type": lib.HCR_E_TYPE, "key": lib.HCR_E_KEY, "unsorted": lib.HCR_E_UNSORTED}
SEG_BOUND = 1024  # HCR_SEG_BOUND of csrc/gvcf_hcr.cuh


def _params(hdr: dict, thr: int, gt: bool, merge: bool):
    from variantcalling_b200.gvcf_hcr import hcr_params

    return hcr_params(VcfHeader("\n".join(D.header(**hdr)) + "\n"), thr, gt, merge)


def _hook(records, hdr=None, thr=20, gt=True, merge=False, seg_bound=0):
    """One hook call against the oracle; returns the hook's result."""
    hdr = hdr or {}
    exp = R.run_text(D.text(records, **hdr), thr, gt, merge)
    body = "".join(r + "\n" for r in records).encode()
    got = lib.test_hcr(body, _params(hdr, thr, gt, merge), seg_bound=seg_bound)
    if "error" in exp:
        assert got.get("error") == (exp["error"][0], REASONS[exp["error"][1]]), (got.get("error"), exp["error"])
        return got
    assert "error" not in got, (got["error"], records[got["error"][0]])
    assert got["bed"].decode() == exp["bed"]
    assert got["skipped"] == exp["skipped"]
    return got


@pytest.mark.parametrize("seg_bound", [0, 1, 2, 5])
def test_hook_crafted(seg_bound):
    for _name, recs in D.crafted_records():
        for thr in (0, 20, 99):
            for gt in (True, False):
                _hook(recs, thr=thr, gt=gt, seg_bound=seg_bound)
            _hook(recs, thr=thr, merge=True, seg_bound=seg_bound)
        _hook(recs, {"gq": "Number=1,Type=Float"}, thr=20, seg_bound=seg_bound)
        _hook(recs, {"info_end": False}, thr=20, seg_bound=seg_bound)


def _no_gq(k):
    """A kept record without GQ (fine under every GQ declaration)."""
    return D.var("chr1", 100 + 10 * k, "A", "C", fmt="GT:DP", sample="0/1:5")


def test_hook_errors():
    pre = [_no_gq(k) for k in range(3)]
    for rec, kind, hdr in D.error_records():
        for gt in (True, False):
            got = _hook(pre + [rec], hdr, gt=gt)
            if kind != "type" or gt:
                assert got.get("error") == (3, REASONS[kind]), (rec, got.get("error"))
        # behind a record that covers it, only the errors that fire before the skip test remain
        got = _hook(["chr1\t400\t.\tA\t<*>\t0\t.\tEND=600\tGT:DP\t0/0:5", rec], hdr)
        assert got.get("error", (None, None))[1] == (None if kind == "type" else REASONS[kind])
    # POS decreasing within a contig
    recs = pre + [D.block("chr1", 101, 101, 30)]
    assert _hook(recs).get("error") == (3, lib.HCR_E_UNSORTED)


def test_hook_random():
    n = int(os.environ.get("UGVC_HCR_RANDOM", "200000"))
    recs = D.random_records(n, 7)
    got = _hook(recs, thr=20)
    assert got["skipped"] > n // 50
    _hook(recs, thr=20, merge=True)
    _hook(recs[: n // 4], thr=0, gt=False)
    _hook(recs[: n // 4], thr=99, seg_bound=3)


@pytest.mark.parametrize("n", [SEG_BOUND // 2, SEG_BOUND + 1, 3 * SEG_BOUND + 17])
def test_hook_alternating(n):
    recs = D.alternating(n)
    got = _hook(recs)
    assert got["longest_segment"] == n
    assert got["skipped"] == n // 2
    _hook(recs, merge=True)
    _hook(recs + [D.block("chr1", 100 + n + 5, 100 + n + 9, 30)] + D.alternating(n, pos0=100 + n + 10), seg_bound=7)


@pytest.mark.parametrize("seg_bound", [0, 4])
def test_hook_entry_state(seg_bound):
    """The kept flags of a piece from the previous piece's exit state: every cut of a record list gives the whole
    list's output."""
    recs = D.random_records(3000, 11, contigs=("chr1", "chr2"), overlap=3.0) + D.alternating(1500, "chr3")
    whole = R.run_text(D.text(recs), 20, True)
    p = _params({}, 20, True, False)
    rng = np.random.default_rng(3)
    for cut in sorted(set(rng.integers(1, len(recs) - 1, 25).tolist()) | {2999, 3000, 3001}):
        a = lib.test_hcr("".join(r + "\n" for r in recs[:cut]).encode(), p, seg_bound=seg_bound)
        cont = recs[cut].split("\t")[0] == recs[cut - 1].split("\t")[0]
        b = lib.test_hcr("".join(r + "\n" for r in recs[cut:]).encode(), p, cont, a["exit_extent"], seg_bound=seg_bound)
        assert (a["bed"] + b["bed"]).decode() == whole["bed"], cut
        assert a["skipped"] + b["skipped"] == whole["skipped"], cut


# ---- the tool, file to file
def _write(tmp_path, records, name="in.g.vcf.gz", **hdr):
    p = str(tmp_path / name)
    bgzf_io.write_vcf_gz(p, D.header(**hdr), records)
    return p


def _tool(path, out, piece=None, merge=False, **kw):
    from variantcalling_b200 import gvcf_hcr as T

    old = T.PIECE_BYTES
    if piece:
        T.PIECE_BYTES = piece
    try:
        if merge:
            return T.gvcf_hcr(path, out, **kw)
        return T.gvcf_to_bed(path, out, **kw)
    finally:
        T.PIECE_BYTES = old


@pytest.fixture(scope="module")
def generated():
    n = int(os.environ.get("UGVC_HCR_FILE_RANDOM", "200000"))
    recs = D.random_records(n, 23, contigs=("chr1", "chr2", "chr3", "chrX"), overlap=2.0)
    # a record whose END covers the rest of chr2, and a stretch without reset points on chr3
    i2 = next(k for k, r in enumerate(recs) if r.startswith("chr2\t")) + 500
    pos = int(recs[i2].split("\t")[1])
    recs[i2] = D.block("chr2", pos, 8_000_000, 40)
    i3 = next(k for k, r in enumerate(recs) if r.startswith("chr3\t"))
    pos = int(recs[i3].split("\t")[1])
    alt = D.alternating(2 * SEG_BOUND + 300, "chr3", pos0=1)
    recs = recs[:i3] + alt + [r for r in recs[i3:] if not r.startswith("chr3\t") or int(r.split("\t")[1]) > len(alt) + 5]
    return recs


@pytest.mark.parametrize("piece", [None, 4096, 150_000])
def test_file_gvcf_to_bed(tmp_path, generated, piece):
    src = _write(tmp_path, generated)
    text = D.text(generated)
    for thr, gt in ((20, True), (0, False), (99, True)):
        out = str(tmp_path / "out.bed")
        skipped = _tool(src, out, piece, gq_threshold=thr, gt=gt)
        exp = R.run_text(text, thr, gt)
        assert open(out).read() == exp["bed"]
        assert skipped == exp["skipped"]


@pytest.mark.parametrize("piece", [None, 4096])
def test_file_gvcf_hcr_merged(tmp_path, generated, piece):
    src = _write(tmp_path, generated)
    out = str(tmp_path / "hcr.bed")
    _tool(src, out, piece, merge=True, gq_threshold=15)
    exp = R.run_text(D.text(generated), 15, True, do_merge=True)
    got = open(out).read()
    assert got == exp["bed"]
    assert got.count("\n") < R.run_text(D.text(generated), 15, True)["bed"].count("\n")


def test_file_crafted_and_empty(tmp_path):
    recs = [r for _n, rs in D.crafted_records() for r in rs]
    recs.sort(key=lambda r: (("chr1", "chr2", "chr3").index(r.split("\t")[0]), int(r.split("\t")[1])))
    src = _write(tmp_path, recs)
    for merge in (False, True):
        out = str(tmp_path / f"c{int(merge)}.bed")
        _tool(src, out, 4096, merge=merge)
        assert open(out).read() == R.run_text(D.text(recs), 20, True, do_merge=merge)["bed"]
    out = str(tmp_path / "empty.bed")
    assert _tool(src, out, gq_threshold=1000) == R.run_text(D.text(recs), 1000)["skipped"]
    assert open(out).read() == ""


def test_file_errors(tmp_path):
    pre = [_no_gq(k) for k in range(3)]
    want = {"type": TypeError, "key": KeyError, "literal": lib.UgvcDataError}
    for k, (rec, kind, hdr) in enumerate(D.error_records()):
        d = tmp_path / str(k)
        d.mkdir()
        src = _write(d, pre + [rec], **hdr)
        with pytest.raises(want[kind], match="record 3 "):
            _tool(src, str(d / "o.bed"))
    # many pieces: the error of a later piece, and one on a skipped record that must not raise
    recs = D.random_records(20000, 5)
    bad_at = 15000
    c, pos = recs[bad_at].split("\t")[:2]
    recs[bad_at] = D.block(c, int(pos), int(pos), ".")
    exp = R.run_text(D.text(recs))
    src = _write(tmp_path, recs, name="late.g.vcf.gz")
    if "error" in exp:
        with pytest.raises(TypeError, match=f"record {exp['error'][0]} "):
            _tool(src, str(tmp_path / "late.bed"), 4096)
    else:
        assert _tool(src, str(tmp_path / "late.bed"), 4096) == exp["skipped"]


def test_file_needs_an_index_and_order(tmp_path):
    recs = [D.block("chr1", 100 + 10 * k, 105 + 10 * k, 30) for k in range(5)]
    src = _write(tmp_path, recs)
    os.remove(src + ".tbi")
    with pytest.raises(ValueError, match="index"):
        _tool(src, str(tmp_path / "o.bed"))
    plain = str(tmp_path / "plain.g.vcf")
    open(plain, "w").write(D.text(recs))
    open(plain + ".tbi", "wb").close()
    with pytest.raises(ValueError, match="index"):
        _tool(plain, str(tmp_path / "o.bed"))
    # contigs that come back, POS decreasing within a contig (across pieces too): ValueError at the record
    many = D.random_records(6000, 9, contigs=("chr1", "chr2"))
    n1 = sum(r.startswith("chr1\t") for r in many)
    for bad, at in ((many + [D.block("chr1", 5, 9, 30)], len(many)),
                    (many[:n1] + [D.block("chr1", 1, 1, 30)] + many[n1:], n1),
                    (many[:4000] + [D.block(many[3999].split("\t")[0], 2, 2, 30)] + many[4000:], 4000)):
        p = str(tmp_path / f"bad{at}.g.vcf.gz")
        w = bgzf_io.BgzfWriter(p)
        w.write(D.text(bad).encode())
        w.close()
        open(p + ".tbi", "wb").close()
        for piece in (None, 4096):
            with pytest.raises(ValueError, match=f"record {at} "):
                _tool(p, str(tmp_path / "o.bed"), piece)


def test_cli(tmp_path, generated):
    import subprocess
    import sys

    src = _write(tmp_path, generated[:30000])
    out = str(tmp_path / "cli.bed")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "ugvc", "__main__.py"), "gvcf_hcr", "--gvcf", src, "--bed", out,
                        "--gq_threshold", "25"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert open(out).read() == R.run_text(D.text(generated[:30000]), 25, True, do_merge=True)["bed"]
    assert "Step 1: Create intervals of high confidence" in r.stderr and "Step 2: Merge intervals" in r.stderr
