"""CPU: the calibrate_bridging_snvs oracle against the reference's own run() and is_homopolymer_snp (golden), the
command line, the output naming and the deviations that are decided before anything is written."""
import gzip
import json
import os

import pytest

from oracle import bridging_snvs_ref as R
from oracle.vcf_reader import OracleHeader
from tests import bridging_snvs_data as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bridging_snvs.json.gz")
RAISES = {"TypeError": TypeError, "ZeroDivisionError": ZeroDivisionError, "KeyError": KeyError, "ValueError": R.FetchError}


def test_oracle_equals_the_reference_golden():
    g = json.load(gzip.open(GOLDEN, "rt"))
    fasta = {k: v.encode("latin-1") for k, v in g["genome"].items()}
    assert fasta == D.genome()
    kinds = {k: R.header_kinds(OracleHeader(D.header(**kw).split("\n"))) for k, kw in g["headers"].items()}
    seen = {"rescued": 0, "walked": 0, **{k: 0 for k in RAISES}}
    assert len(g["entries"]) > 30000
    for line, hkey, args, want, hm in g["entries"]:
        m, q, tv, nv, nd, edge, set_qual = args
        call = (line, kinds[hkey], fasta, m, q, tv, nv, nd, edge)
        if isinstance(want, str):
            with pytest.raises(RAISES[want]):
                R.decide(*call)
            seen[want] += 1
            continue
        rescued, hmer, seq = R.decide(*call)
        cols = line.split("\t")
        if rescued:
            seen["rescued"] += 1
            assert want["logs"] == [f"refseq : {seq} hmer_size: {hmer}", line + "\n"], line
            assert (want["qual"], want["filter"]) == (set_qual, ["PASS"])
        else:
            assert want["logs"] == [], line
            assert want["filter"] == ([] if cols[6] == "." else cols[6].split(";"))
        # is_homopolymer_snp alone: the candidate test, the walk and the qualifying test
        if isinstance(hm, str):
            continue
        ok, info = hm
        if info == "not a filtered snp above min_qual":
            assert (ok, hmer) == (False, 0), line
        else:
            seen["walked"] += 1
            assert info.startswith("refseq : " if ok else f"hmer_size: {hmer} "), (line, info, hmer)
            if ok:
                assert info == f"refseq : {seq} hmer_size: {hmer}"
    assert all(v > 0 for v in seen.values()), seen


def test_window_edges():
    g = {"c": b"AAAAACGTTTTT"}
    kinds = R.header_kinds(OracleHeader(D.header().split("\n")))
    # m = 0: the upstream walk starts at the variant's own reference base
    r, h, seq = R.decide(D.rec("c", 6, "C", "A"), kinds, g, 0)
    assert (h, seq) == (1, "C")
    # a window past the contig's end is clipped; a start at or past the end reads empty
    assert R.decide(D.rec("c", 12, "T", "T"), kinds, g, 3)[2] == "TTTT"
    assert R.decide(D.rec("c", 20, "T", "T"), kinds, g, 3)[1:] == (1, "")
    with pytest.raises(R.FetchError):
        R.decide(D.rec("c", 3, "A", "A"), kinds, g, 3)
    with pytest.raises(R.FetchError):
        R.decide(D.rec("d", 10, "A", "A"), kinds, g, 3)


def test_cli_parsing_and_params():
    from ugvc.__main__ import TOOLS
    from variantcalling_b200 import bridging_snvs as T
    from variantcalling_b200 import lib
    from variantcalling_b200.vcf_header import VcfHeader

    assert TOOLS["calibrate_bridging_snvs"] == "variantcalling_b200.bridging_snvs"
    a = T.parse_args(["--vcf", "i.vcf.gz", "--reference", "r.fa", "--output", "o.vcf.gz"])
    assert (a.min_query_hmer_size, a.min_initial_qual, a.min_tumor_vaf, a.max_normal_vaf, a.min_normal_depth,
            a.min_distance_from_edge, a.set_qual, a.device) == (5, 5, 0.2, 0.1, 10, 0, 20, None)
    with pytest.raises(SystemExit):
        T.parse_args(["--vcf", "i.vcf.gz", "--output", "o"])
    hdr = VcfHeader(D.header())
    p = T.bsn_params(hdr, set_qual=37)
    assert (p.qual_text, p.ad_kind, p.ad_integer, p.dp_kind) == (b"37", lib.BSN_KIND_TUPLE, 1, lib.BSN_KIND_SCALAR)
    assert T.qual_text(20) == R.qual_text(20).encode() == b"20"
    assert T.qual_text(123456789) == R.qual_text(123456789).encode() == b"1.23457e+08"
    assert T.bsn_params(VcfHeader(D.header(bg_ad=None))).bg_ad_kind == lib.BSN_KIND_NONE
    for key in ("ad", "dp", "bg_ad", "bg_dp"):
        with pytest.raises(NotImplementedError):
            T.bsn_params(VcfHeader(D.header(**{key: "Number=1,Type=String"})))
    with pytest.raises(ValueError, match="min_query_hmer_size"):
        T.bsn_params(hdr, min_query_hmer_size=-1)


def test_fasta_loading(tmp_path):
    from variantcalling_b200 import bridging_snvs as T
    from variantcalling_b200 import bgzf_io

    g = D.genome()
    ref = str(tmp_path / "ref.fa")
    with open(ref, "wb") as fh:
        for name, seq in g.items():
            fh.write(b">" + name.encode() + b" x\n" + b"\n".join(seq[k: k + 50] for k in range(0, len(seq), 50)) + b"\n")
    vcf = str(tmp_path / "in.vcf.gz")
    text = D.text([D.rec("chr2", 100, "A", "C"), D.rec("chrZ", 100, "A", "C")], contigs=("chr2", "chrZ"))
    open(vcf, "w").write(text)
    assert T.load_contigs(ref, vcf) == g  # no index: every FASTA contig
    hl = [ln for ln in text.split("\n") if ln.startswith("#")]
    bgzf_io.write_vcf_gz(vcf, hl, [ln for ln in text.split("\n") if ln and not ln.startswith("#")])
    assert T.load_contigs(ref, vcf) == {"chr2": g["chr2"]}  # the contigs the .tbi names that the FASTA holds
