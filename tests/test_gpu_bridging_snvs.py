"""GPU: calibrate_bridging_snvs on the device against oracle/bridging_snvs_ref.py -- output text byte for byte, valid BGZF
blocks, the .tbi read back by oracle/tabix_ref.py, the rescued count, the log lines and the error contract, for plain
text, BGZF with and without .tbi, output names with and without .gz, several pieces and a contig missing from the FASTA.
The test_hook_* tests run the kernels alone (ugvc_test_bsn) and also run on the host emulation
(tests/test_bridging_snvs_emu_cpu.py)."""
import gzip
import logging
import os

import numpy as np
import pytest

from oracle import bridging_snvs_ref as R
from oracle import tabix_ref as TR
from tests import bridging_snvs_data as D
from variantcalling_b200 import bgzf_io, lib

pytestmark = pytest.mark.gpu

G = D.genome()
REASONS = {"literal": lib.BSN_E_LITERAL, "type": lib.BSN_E_TYPE, "zero": lib.BSN_E_ZERO_DIVISION, "key": lib.BSN_E_KEY,
           "fetch": lib.BSN_E_FETCH}


def _hook_once(records, hdr, fasta, **kw):
    """One hook call against the oracle; returns the record index of the error both raise at, or None."""
    text = D.text(records, **hdr)
    exp = R.run_text(text, fasta, **kw)
    body = "".join(r + "\n" for r in records).encode()
    got = lib.test_bsn(body, fasta, D.params(D.header(**hdr), **kw))
    if "error" in exp:
        assert got.get("error") == (exp["error"][0], REASONS[exp["error"][1]]), (got, exp["error"], records[exp["error"][0]])
        return exp["error"][0]
    assert "error" not in got, (got, records[got["error"][0]])
    assert got["text"].decode() == "".join(r + "\n" for r in exp["records"])
    assert got["rescued"].tolist() == exp["rescued"] and got["n_rescued"] == exp["n_rescued"]
    assert got["hmer"].tolist() == exp["hmer"]
    want_end = [int(r.split("\t")[7][4:]) if r.split("\t")[7].startswith("END=") else 0 for r in exp["records"]]
    assert got["end"].tolist() == want_end
    return None


def _hook(records, hdr=None, fasta=G, **kw):
    """Every record checked: after an error the records up to it are dropped and the rest run again."""
    hdr = hdr or {}
    n_err = 0
    while records:
        at = _hook_once(records, hdr, fasta, **kw)
        if at is None:
            break
        n_err += 1
        records = records[at + 1:]
    return n_err


@pytest.mark.parametrize("m", [0, 1, 2, 3, 4, 5, 6])
def test_hook_crafted(m):
    recs = D.crafted_records(G)
    for edge in (0, 1, 2):
        _hook(recs, min_query_hmer_size=m, min_distance_from_edge=edge)
    _hook(recs, {"dp": "Number=1,Type=Float", "bg_dp": "Number=1,Type=Float", "ad": "Number=.,Type=Float"},
          min_query_hmer_size=m, min_initial_qual=4.9, set_qual=37)
    _hook(recs, {"ad": "Number=1,Type=Integer", "bg_dp": "Number=A,Type=Integer"}, min_query_hmer_size=m)
    _hook(recs, {"bg_ad": None}, min_query_hmer_size=m, min_tumor_vaf=0.5, max_normal_vaf=0.0, min_normal_depth=0)


def test_hook_errors():
    for rec, kind in D.error_records(G):
        recs = [D.rec("chr1", 100 + k, "A", "C", flt="PASS") for k in range(3)] + [rec]
        exp = R.run_text(D.text(recs), G)
        assert exp["error"] == (3, kind), (rec, exp)
        _hook_once(recs, {}, G)
    # undeclared keys raise KeyError only where the rescue reads them
    pos, ref, alt = D.hmer_sites(G, "chr1", 5)[0]
    recs = [D.rec("chr1", pos, ref, alt, flt="PASS"), D.rec("chr1", pos, ref, alt)]
    assert R.run_text(D.text(recs, bg_dp=None), G)["error"] == (1, "key")
    _hook_once(recs, {"bg_dp": None}, G)
    # a Number=1 AD: a slice of a scalar
    recs = [D.rec("chr1", pos, ref, alt, s0="0/1:8:18:20,0:20")]
    assert R.run_text(D.text(recs, ad="Number=1,Type=Integer"), G)["error"] == (0, "type")
    _hook_once(recs, {"ad": "Number=1,Type=Integer"}, G)


def test_hook_random():
    n = int(os.environ.get("UGVC_BSN_RANDOM", "100000"))
    recs = D.random_records(G, n, 31)
    for m in (3, 5):
        assert _hook(recs, min_query_hmer_size=m) == 0
    assert sum(R.run_text(D.text(recs), G)["rescued"]) > n // 100


# ---- the tool, file to file
def _write_input(tmp_path, text, form):
    p = str(tmp_path / "in.vcf.gz")
    if form == "text":
        open(p, "w").write(text)
        return p
    hl = [ln for ln in text.split("\n") if ln.startswith("#")]
    rl = [ln for ln in text.split("\n") if ln and not ln.startswith("#")]
    bgzf_io.write_vcf_gz(p, hl, rl)
    if form == "bgzf":
        os.remove(p + ".tbi")
    return p


def _write_fasta(tmp_path, fasta, fai):
    p = str(tmp_path / "ref.fa")
    with open(p, "wb") as fh:
        offs = []
        for name, seq in fasta.items():
            fh.write(b">" + name.encode() + b" desc\n")
            offs.append((name, len(seq), fh.tell()))
            for k in range(0, len(seq), 60):
                fh.write(seq[k: k + 60] + b"\n")
    if fai:
        with open(p + ".fai", "w") as fh:
            for name, n, off in offs:
                fh.write(f"{name}\t{n}\t{off}\t60\t61\n")
    return p


def _run_tool(tmp_path, text, form, fasta=G, gz=True, piece=None, fai=True, **kw):
    from variantcalling_b200 import bridging_snvs as T

    src = _write_input(tmp_path, text, form)
    ref = _write_fasta(tmp_path, fasta, fai)
    out = str(tmp_path / ("out.vcf.gz" if gz else "out.vcf"))
    old = T.PIECE_BYTES
    if piece:
        T.PIECE_BYTES = piece
    try:
        n = T.calibrate_bridging_snvs(src, ref, out, **kw)
    finally:
        T.PIECE_BYTES = old
    return (out if gz else out + ".gz"), n


def _check_output(path, n_rescued, exp):
    TR.read_bgzf_blocks(path)  # every block valid for zlib, CRC32 / ISIZE right, EOF block present
    got = gzip.open(path, "rt").read()
    assert got == "\n".join(exp["header"]) + "\n" + "".join(r + "\n" for r in exp["records"])
    assert n_rescued == exp["n_rescued"]
    idx = TR.TabixIndex(path + ".tbi")
    ivs = []
    for r in exp["records"]:
        c = r.split("\t")
        ivs.append((c[0], int(c[1]) - 1, int(c[1]) - 1 + len(c[3])))
        if c[7].startswith("END=") and int(c[7][4:]) > ivs[-1][1]:
            ivs[-1] = (c[0], ivs[-1][1], int(c[7][4:]))
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
        want = {recs[j] for j, (c2, b2, e2) in enumerate(ivs) if c2 == c and b2 < e and e2 > b}
        assert sorted(hits) == sorted(want)  # the reader reports a repeated line once


def _logs(caplog):
    return [r.getMessage() for r in caplog.records if r.name == "variantcalling_b200.bridging_snvs"]


@pytest.mark.parametrize("form", ["text", "bgzf_tbi", "bgzf"])
@pytest.mark.parametrize("gz", [True, False])
def test_crafted_file(tmp_path, form, gz, caplog):
    caplog.set_level(logging.INFO)
    recs = [r for r in D.crafted_records(G) if "error" not in R.run_text(D.text([r]), G, min_query_hmer_size=3)]
    recs.sort(key=lambda r: (("chr1", "chr2", "chrM").index(r.split("\t")[0]), int(r.split("\t")[1])))
    text = D.text(recs)
    exp = R.run_text(text, G, min_query_hmer_size=3)
    assert exp["n_rescued"] > 10
    out, n = _run_tool(tmp_path, text, form, gz=gz, fai=form != "bgzf", min_query_hmer_size=3)
    _check_output(out, n, exp)
    assert _logs(caplog) == exp["logs"]


@pytest.fixture(scope="module")
def five_contigs():
    """Random records over five contigs, one of them (chrX) missing from the FASTA and never a candidate."""
    g = D.genome(11, (("chr1", 40000), ("chr2", 30000), ("chr3", 20000), ("chr10", 20000), ("chrX", 5000)))
    contigs = ("chr1", "chr2", "chr3", "chr10", "chrX")
    n = int(os.environ.get("UGVC_BSN_FILE_RANDOM", "300000"))
    recs = D.random_records(g, n, 41, contigs=contigs)
    recs = [r if not r.startswith("chrX\t") else "\t".join(r.split("\t")[:6] + ["PASS"] + r.split("\t")[7:]) for r in recs]
    fasta = {c: g[c] for c in contigs if c != "chrX"}
    text = D.text(recs, contigs=contigs)
    return text, fasta, R.run_text(text, fasta)


@pytest.mark.parametrize("form", ["text", "bgzf_tbi", "bgzf"])
def test_five_contigs_pieces(tmp_path, form, five_contigs, caplog):
    caplog.set_level(logging.INFO)
    text, fasta, exp = five_contigs
    assert "error" not in exp and exp["n_rescued"] > 100
    out, n = _run_tool(tmp_path, text, form, fasta=fasta, piece=2 << 20)
    _check_output(out, n, exp)
    assert _logs(caplog) == exp["logs"]


def test_errors_on_the_file_path(tmp_path):
    from variantcalling_b200 import bridging_snvs as T

    for k, (rec, kind) in enumerate(D.error_records(G)):
        d = tmp_path / str(k)
        d.mkdir()
        recs = [D.rec("chr1", 100 + j, "A", "C", flt="PASS") for j in range(3)] + [rec]
        want = {"type": TypeError, "zero": ZeroDivisionError, "key": KeyError, "fetch": ValueError,
                "literal": lib.UgvcDataError}[kind]
        with pytest.raises(want, match="record 3"):
            _run_tool(d, D.text(recs), "bgzf" if k % 2 else "text")
    with pytest.raises(NotImplementedError):
        _run_tool(tmp_path, D.text([], dp="Number=1,Type=String"), "text")
    with pytest.raises(ValueError, match="min_query_hmer_size"):
        _run_tool(tmp_path, D.text([]), "text", min_query_hmer_size=-1)
    assert T.qual_text(20) == b"20"


def test_cli(tmp_path, caplog):
    import subprocess
    import sys

    recs = [D.rec("chr1", p, r, a) for p, r, a in D.hmer_sites(G, "chr1", 5)[:20]]
    text = D.text(recs)
    src = _write_input(tmp_path, text, "bgzf_tbi")
    ref = _write_fasta(tmp_path, G, True)
    out = str(tmp_path / "cli.vcf")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "ugvc", "__main__.py"), "calibrate_bridging_snvs", "--vcf", src,
                        "--reference", ref, "--output", out, "--set_qual", "33"], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    exp = R.run_text(text, G, set_qual=33)
    assert exp["n_rescued"] > 0
    _check_output(out + ".gz", exp["n_rescued"], exp)
    for line in exp["logs"]:
        assert line.rstrip("\n") in r.stderr
