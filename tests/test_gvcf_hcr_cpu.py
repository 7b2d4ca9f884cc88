"""CPU: gvcf_hcr's oracle pinned to the reference's own gvcf_to_bed (tests/golden/gvcf_hcr.json.gz,
scripts/make_golden_gvcf_hcr.py), the host's join of merged lines across pieces, the kernels' parameters, the command
line, the dispatcher entry and the index requirement."""
import gzip
import json
import os

import numpy as np
import pytest

from oracle import gvcf_hcr_ref as R
from tests import gvcf_hcr_data as D
from variantcalling_b200 import bgzf_io, lib
from variantcalling_b200 import gvcf_hcr as T
from variantcalling_b200.vcf_header import VcfHeader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    with gzip.open(os.path.join(ROOT, "tests", "golden", "gvcf_hcr.json.gz"), "rt") as fh:
        return json.load(fh)["cases"]


def test_oracle_matches_the_reference():
    cases = _golden()
    kinds = set()
    for c in cases:
        got = R.run_text(c["text"], c["gq_threshold"], c["gt"])
        want = c["result"]
        if "error" in want:
            kinds.add(want["error"][1])
            assert got.get("error") == tuple(want["error"]), c["name"]
        else:
            assert got == {"bed": want["bed"], "skipped": want["skipped"]}, c["name"]
    assert kinds == {"type", "key", "literal"}
    assert sum(c["result"].get("skipped", 0) for c in cases) > 1000
    names = {c["name"] for c in cases}
    assert {"refcall_gts", "long_deletion", "gq_on_skipped", "book_ended_and_gapped", "alternating"} <= names


def test_merge_rule():
    ivs = [("a", 0, 5), ("a", 5, 9), ("a", 10, 12), ("a", 11, 20), ("b", 20, 30), ("b", 30, 31)]
    assert R.merge(ivs) == [("a", 0, 9), ("a", 10, 20), ("b", 20, 31)]


def test_join_across_pieces():
    """Merging each piece's selected intervals and joining the pieces gives the merge of the whole, for every cut."""
    recs = D.random_records(4000, 3, overlap=0.2)
    ivs, _ = R.gvcf_to_bed_records(R.iterate(D.text(recs)), 10, True)
    whole = R.bed_text(R.merge(ivs)).encode()
    rng = np.random.default_rng(1)
    for n_cuts in (1, 2, 7, 40):
        cuts = sorted(set(rng.integers(0, len(ivs), n_cuts).tolist()))
        parts = [ivs[a:b] for a, b in zip([0, *cuts], [*cuts, len(ivs)])]
        held, out = b"", b""
        for p in parts:
            now, held = T.join_pieces(held, R.bed_text(R.merge(p)).encode())
            out += now
        assert out + held == whole, cuts
    assert T.join_pieces(b"", b"") == (b"", b"")
    assert T.join_pieces(b"c\t1\t5\n", b"") == (b"", b"c\t1\t5\n")


@pytest.mark.parametrize("decl,kind,integer", [("Number=1,Type=Integer", lib.HCR_GQ_SCALAR, 1),
                                               ("Number=1,Type=Float", lib.HCR_GQ_SCALAR, 0),
                                               ("Number=.,Type=Integer", lib.HCR_GQ_TUPLE, 1),
                                               ("Number=1,Type=String", lib.HCR_GQ_STRING, 0),
                                               (None, lib.HCR_GQ_STRING, 0)])
def test_params(decl, kind, integer):
    for info_end in (True, False):
        h = VcfHeader("\n".join(D.header(gq=decl, info_end=info_end)) + "\n")
        p = T.hcr_params(h, 17, False, True)
        assert (p.gq_threshold, p.gt, p.merge, p.info_end, p.gq_kind, p.gq_integer) == (17, 0, 1, int(info_end), kind, integer)


def test_cli_and_dispatcher():
    a = T.parse_args(["--gvcf", "x.g.vcf.gz", "--bed", "o.bed"])
    assert (a.gvcf, a.bed, a.gq_threshold, a.device) == ("x.g.vcf.gz", "o.bed", 20, None)
    assert T.parse_args(["--gvcf", "x", "--bed", "o", "--gq_threshold", "7"]).gq_threshold == 7
    import importlib.util

    spec = importlib.util.spec_from_file_location("ugvc_main", os.path.join(ROOT, "ugvc", "__main__.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    assert m.TOOLS["gvcf_hcr"] == "variantcalling_b200.gvcf_hcr"


def test_an_index_is_required(tmp_path):
    recs = [D.block("chr1", 100 + 10 * k, 105 + 10 * k, 30) for k in range(5)]
    src = str(tmp_path / "in.g.vcf.gz")
    bgzf_io.write_vcf_gz(src, D.header(), recs)
    os.remove(src + ".tbi")
    with pytest.raises(ValueError, match="index"):
        T.gvcf_to_bed(src, str(tmp_path / "o.bed"))
    plain = str(tmp_path / "plain.g.vcf")
    open(plain, "w").write(D.text(recs))
    open(plain + ".tbi", "wb").close()
    with pytest.raises(ValueError, match="index"):
        T.gvcf_hcr(plain, str(tmp_path / "o.bed"))
