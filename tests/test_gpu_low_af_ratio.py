"""GPU: filter_low_af_ratio_to_background on the device against oracle/low_af_ratio_ref.py -- output text byte for
byte, valid BGZF blocks, the .tbi read back by oracle/tabix_ref.py, the filtered count and the error contract, for plain
text, BGZF with and without .tbi, and output names with and without .gz.  The test_hook_* tests run the kernels alone
(ugvc_test_afr) and also run on the host emulation (tests/test_low_af_ratio_emu_cpu.py)."""
import gzip
import logging
import os

import numpy as np
import pytest

from oracle import low_af_ratio_ref as R
from oracle import tabix_ref as TR
from tests import low_af_ratio_data as D
from variantcalling_b200 import bgzf_io, lib

pytestmark = pytest.mark.gpu


def _split(text):
    lines = text.split("\n")
    head = "".join(ln + "\n" for ln in lines if ln.startswith("#"))
    body = "".join(ln + "\n" for ln in lines if ln and not ln.startswith("#"))
    return head, body


def _hook(text, **kw):
    head, body = _split(text)
    exp = R.run_text(text, **kw)
    got = lib.test_afr(body.encode(), D.params(head, **kw))
    if "error" in exp:
        assert got.get("error") == (exp["error"][0], {"literal": lib.AFR_E_LITERAL, "type": lib.AFR_E_TYPE}[exp["error"][1]])
        return
    assert "error" not in got, got
    assert got["text"].decode() == "".join(r + "\n" for r in exp["records"])
    assert got["failed"].tolist() == exp["failed"] and got["n_filtered"] == exp["n_filtered"]
    want_end = []
    for r in exp["records"]:
        v = 0
        for kv in ([] if r.split("\t")[7] == "." else r.split("\t")[7].split(";")):
            if kv.startswith("END="):
                v = int(kv[4:]) if kv[4:].isdigit() and len(kv) <= 14 else 0  # noqa: PLR2004
                break
        want_end.append(v)
    assert got["end"].tolist() == want_end


@pytest.mark.parametrize("hdr", [{}, {"vaf": "Number=1,Type=Float"}, {"bg": "Number=.,Type=Integer"},
                                 {"vt": "Number=.,Type=String"}, {"vaf": ""}, {"vt": None}])
@pytest.mark.parametrize("thr", [(10, 0, 0), (10, 2, 0.15), (2, 1, 0.3)])
def test_hook_crafted(hdr, thr):
    for nf in ("LowAFRatioToBackground", "MyCustomFilter"):
        _hook(D.crafted_text(**hdr), af_ratio_threshold=thr[0], af_ratio_threshold_h_indels=thr[1], t_vaf_threshold=thr[2],
              new_filter=nf)


def test_hook_unit_and_random():
    _hook(D.unit_text(), af_ratio_threshold=10, af_ratio_threshold_h_indels=2, t_vaf_threshold=0.15)
    n = int(os.environ.get("UGVC_AFR_RANDOM", "100000"))
    _hook(D.random_text(n, 3, 11), af_ratio_threshold=10, af_ratio_threshold_h_indels=2, t_vaf_threshold=0.15)
    _hook(D.random_text(n // 10, 5, 12, vaf="Number=R,Type=Float"), af_ratio_threshold=3)


def test_hook_literal_errors():
    base = D.header(2)
    rec = "chr1\t{p}\t.\tA\tT\t.\tPASS\tVARIANT_TYPE=snp\tGT:VAF:BG_VAF\t0/1:0.5:0.4\t{s}"
    for bad in ("0/1:0.5x:0.4", "0/1:0.5:1e", "a/1:0.5:0.4", "0/1:0.5,:0.4", "0/1:1.5.2:0.4"):
        text = base + "".join(rec.format(p=100 + k, s="0/1:0.5:0.4") + "\n" for k in range(3)) + rec.format(p=200, s=bad) + "\n"
        _hook(text)
        assert R.run_text(text)["error"] == (3, "literal")
    # Number=1 VAF: TypeError at the first record that reaches an alt allele, not at a RefCall or hom-ref record
    text = D.header(1, vaf="Number=1,Type=Float") + "".join(
        "\t".join(["chr1", str(100 + k), ".", "A", "T", ".", flt, ".", "GT:VAF:BG_VAF", gt]) + "\n"
        for k, (flt, gt) in enumerate([("RefCall", "0/1:0.5:0.4"), ("PASS", "0/0:0.5:0.4"), ("PASS", "0/1:.:0.4"),
                                       ("PASS", "0/1:0.5:0.4")]))
    assert R.run_text(text)["error"] == (3, "type")
    _hook(text)


# ---- the tool, file to file
def _write_input(tmp_path, text, form):
    if form == "text":
        p = str(tmp_path / "in.vcf.gz")  # plain text under a .gz name, as the reference's unit test writes it
        open(p, "w").write(text)
        return p
    p = str(tmp_path / "in.vcf.gz")
    head, body = _split(text)
    hl, rl = head.rstrip("\n").split("\n"), body.rstrip("\n").split("\n") if body else []
    bgzf_io.write_vcf_gz(p, hl, rl)
    if form == "bgzf":
        os.remove(p + ".tbi")
    return p


def _run_tool(tmp_path, text, form, gz=True, piece=None, **kw):
    from variantcalling_b200 import low_af_ratio as T

    src = _write_input(tmp_path, text, form)
    out = str(tmp_path / ("out.vcf.gz" if gz else "out.vcf"))
    old = T.PIECE_BYTES
    if piece:
        T.PIECE_BYTES = piece
    try:
        T.filter_low_af_ratio_to_background(src, out, **kw)
    finally:
        T.PIECE_BYTES = old
    return out if gz else out + ".gz"


def _check_output(path, text, exp=None, **kw):
    exp = exp or R.run_text(text, **kw)
    TR.read_bgzf_blocks(path)  # every block valid for zlib, CRC32 / ISIZE right, EOF block present
    got = gzip.open(path, "rt").read()
    want = "\n".join(exp["header"]) + "\n" + "".join(r + "\n" for r in exp["records"])
    assert got == want
    idx = TR.TabixIndex(path + ".tbi")
    ivs = R.intervals(exp["records"], True)
    names = []
    for c, _b, _e in ivs:
        if not names or names[-1] != c:
            names.append(c)
    assert idx.names == names
    rng = np.random.default_rng(5)
    recs = [r.encode() for r in exp["records"]]
    for k in rng.choice(len(ivs), size=min(40, len(ivs)), replace=False) if ivs else []:
        c, b, e = ivs[k]
        hits = TR.query(path, idx, c, b, e)
        want_hits = sorted((recs[j] for j, (c2, b2, e2) in enumerate(ivs) if c2 == c and b2 < e and e2 > b),
                           key=lambda ln: int(ln.split(b"\t")[1]))
        assert sorted(hits) == sorted(want_hits)
    return exp


@pytest.mark.parametrize("form", ["text", "bgzf_tbi", "bgzf"])
@pytest.mark.parametrize("gz", [True, False])
def test_unit_scenarios(tmp_path, form, gz, caplog):
    text = D.unit_text()
    caplog.set_level(logging.INFO)
    for k, (kw, flagged) in enumerate([
            (dict(af_ratio_threshold=10, af_ratio_threshold_h_indels=2, t_vaf_threshold=0.15), [0, 1, 3, 5, 7, 9]),
            (dict(af_ratio_threshold=0.05, af_ratio_threshold_h_indels=0.05, t_vaf_threshold=1), []),
            (dict(af_ratio_threshold=10, af_ratio_threshold_h_indels=2, t_vaf_threshold=0.5, new_filter="MyCustomFilter"),
             None)]):
        d = tmp_path / str(k)
        d.mkdir()
        out = _run_tool(d, text, form, gz, **kw)
        exp = _check_output(out, text, **kw)
        nf = kw.get("new_filter", "LowAFRatioToBackground")
        got = [i for i, r in enumerate(gzip.open(out, "rt").read().split("\n")) if r and not r.startswith("#")]
        recs = [r for r in gzip.open(out, "rt").read().split("\n") if r and not r.startswith("#")]
        marked = [i for i, r in enumerate(recs) if nf in r.split("\t")[6].split(";")]
        if flagged is not None:
            assert marked == flagged
        else:
            assert marked[:2] == [0, 1]
        assert recs[2].split("\t")[6] == "RefCall"
        assert f"Filtered {exp['n_filtered']} variants with {nf} filter." in caplog.text
        assert len(got) == 10


@pytest.mark.parametrize("form", ["text", "bgzf_tbi", "bgzf"])
def test_crafted_file(tmp_path, form):
    for k, hdr in enumerate([{}, {"vaf": "Number=R,Type=Float"}, {"vt": "Number=.,Type=String"},
                             {"extra": ('##FILTER=<ID=LowAFRatioToBackground,Description="old">',)}]):
        d = tmp_path / str(k)
        d.mkdir()
        text = D.crafted_text(**hdr)
        _check_output(_run_tool(d, text, form, gz=k % 2 == 0), text)


RANDOM_KW = dict(af_ratio_threshold=5, af_ratio_threshold_h_indels=2, t_vaf_threshold=0.2)


@pytest.fixture(scope="module")
def random_1m():
    n = int(os.environ.get("UGVC_AFR_FILE_RANDOM", "1000000"))
    text = D.random_text(n, 2, 21, contigs=("chr1", "chr2", "chr3", "chr10", "chrX"))
    return text, R.run_text(text, **RANDOM_KW)


@pytest.mark.parametrize("form", ["text", "bgzf_tbi", "bgzf"])
def test_random_1m_pieces(tmp_path, form, random_1m):
    text, exp = random_1m
    _check_output(_run_tool(tmp_path, text, form, piece=8 << 20, **RANDOM_KW), text, exp, **RANDOM_KW)


def test_errors_on_the_file_path(tmp_path):
    from variantcalling_b200 import low_af_ratio as T

    text = D.header(1, vaf="Number=1,Type=Float") + "chr1\t100\t.\tA\tT\t.\tPASS\t.\tGT:VAF:BG_VAF\t0/1:0.5:0.4\n"
    with pytest.raises(TypeError):
        _run_tool(tmp_path, text, "bgzf")
    text = D.header(1) + "chr1\t100\t.\tA\tT\t.\tPASS\t.\tGT:VAF:BG_VAF\t0/1:0.5q:0.4\n"
    with pytest.raises(lib.UgvcDataError):
        _run_tool(tmp_path, text, "text")
    with pytest.raises(NotImplementedError):
        _run_tool(tmp_path, D.header(1, vaf="Number=A,Type=String"), "text")
    for bad in ("A;B", "PASS", "RefCall", "a b", "x=y", ""):
        with pytest.raises(ValueError):
            T.filter_low_af_ratio_to_background(_write_input(tmp_path, D.unit_text(), "text"), str(tmp_path / "o.vcf.gz"),
                                                new_filter=bad)
    text = D.header(1) + "chr1\t100\t.\tA\tT\t.\tPASS\t.\tGT\t0/1\nchr2\t100\t.\tA\tT\t.\tPASS\t.\tGT\t0/1\n" \
        "chr1\t200\t.\tA\tT\t.\tPASS\t.\tGT\t0/1\n"
    with pytest.raises(ValueError, match="contiguous"):
        _run_tool(tmp_path, text, "text")


def test_cli(tmp_path):
    import subprocess
    import sys

    src = _write_input(tmp_path, D.unit_text(), "bgzf_tbi")
    out = str(tmp_path / "cli.vcf.gz")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "ugvc", "__main__.py"), "filter_low_af_ratio_to_background", src, out,
                        "--af_ratio_threshold", "10", "--af_ratio_threshold_h_indels", "2", "--tumor_vaf_threshold_h_indels",
                        "0.15"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    recs = [ln for ln in gzip.open(out, "rt").read().split("\n") if ln and not ln.startswith("#")]
    assert [i + 1 for i, ln in enumerate(recs) if "LowAFRatioToBackground" in ln.split("\t")[6]] == [1, 2, 4, 6, 8, 10]
    assert recs[2].split("\t")[6] == "RefCall"
    assert "For snps and non-h-indels: 10.0, and for h-indels (applied only if tumor VAF<0.15: 2.0)" in gzip.open(out, "rt").read()
