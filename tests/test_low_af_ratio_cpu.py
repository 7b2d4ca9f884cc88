"""CPU: the filter_low_af_ratio_to_background oracle against the reference's own process_record (golden), the FILTER
edit of htslib's bcf_add_filter on crafted lists, the header text and the command line."""
import gzip
import json
import os

import pytest

from oracle import low_af_ratio_ref as R
from oracle.vcf_reader import OracleHeader
from tests import low_af_ratio_data as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "low_af_ratio.json.gz")


def test_oracle_equals_the_reference_golden():
    g = json.load(gzip.open(GOLDEN, "rt"))
    kinds = {k: R.header_kinds(OracleHeader(D.header(1, **kw).split("\n"))) for k, kw in g["headers"].items()}
    kinds["unit"] = R.header_kinds(OracleHeader(D.unit_text().split("\n")))
    n_type = 0
    assert len(g["entries"]) > 10000
    for line, hkey, thr, want in g["entries"]:
        try:
            out, failed = R.edit_record(line, kinds[hkey], *thr)
        except TypeError:
            assert want == "TypeError", line
            n_type += 1
            continue
        refcall = "RefCall" in line.split("\t")[6].split(";")
        assert failed == (want is True and not refcall), (line, thr, want)
    assert n_type > 0


def test_unit_decisions():
    text = D.unit_text()
    res = R.run_text(text, af_ratio_threshold=10, af_ratio_threshold_h_indels=2, t_vaf_threshold=0.15)
    assert [i + 1 for i, f in enumerate(res["failed"]) if f] == [1, 2, 4, 6, 8, 10]
    assert res["records"][2] == [ln for ln in text.split("\n") if "RefCall\tVARIANT" in ln][0]  # untouched
    assert R.run_text(text, af_ratio_threshold=0.05, af_ratio_threshold_h_indels=0.05, t_vaf_threshold=1)["n_filtered"] == 0


@pytest.mark.parametrize("flt, failed, want", [
    (".", True, "NF"), (".", False, "."), ("PASS", True, "NF"), ("PASS", False, "PASS"),
    ("A", True, "A;NF"), ("A;A", True, "A;A;NF"), ("A;A", False, "A;A"), ("PASS;A", True, "PASS;A;NF"),
    ("NF", False, "."), ("NF", True, "NF"), ("NF;A", False, "A"), ("A;NF", True, "A;NF"), ("A;NF;B", False, "A;B"),
    ("NF;A;NF;A", False, "A"), ("A;NF;A;B", True, "A;B;NF"), ("PASS;NF", False, "PASS"), ("PASS;NF", True, "NF"),
    ("A;NF;PASS", False, "PASS"), ("A;NF;PASS;B", True, "B;NF"), ("PASS;NF;PASS", False, "PASS"),
    ("RefCall;NF", True, "RefCall;NF"), ("A;RefCall", True, "A;RefCall")])
def test_filter_edit(flt, failed, want):
    kinds = {"VARIANT_TYPE": True, "VAF": ("A", "Float"), "BG_VAF": ("A", "Float")}
    sample = "0/1:0.5:0.01" if not failed else "0/1:0.5:0.5"
    line = "\t".join(["chr1", "1", ".", "A", "T", ".", flt, ".", "GT:VAF:BG_VAF", sample])
    out, f = R.edit_record(line, kinds, new_filter="NF")
    assert out.split("\t")[6] == want
    assert f == (failed and "RefCall" not in flt)


def test_header_text():
    from variantcalling_b200 import low_af_ratio as T
    from variantcalling_b200.vcf_header import VcfHeader

    text = D.unit_text()
    hdr = VcfHeader(text)
    lines = T.output_lines(hdr, "LowAFRatioToBackground", T.filter_description(10, 0, 0))
    exp = R.run_text(text)["header"]
    assert lines == exp
    assert '##FILTER=<ID=LowAFRatioToBackground,Description="Filter variants if AF ratio to background in GT ALT alleles ' \
           '< threshold. For snps and non-h-indels: 10, and for h-indels (applied only if tumor VAF<0: 0)">' in lines
    assert lines[1] == '##FILTER=<ID=PASS,Description="All filters passed">'
    assert lines[-2].startswith("##FILTER=<ID=LowAFRatioToBackground")
    declared = VcfHeader(D.header(1, extra=('##FILTER=<ID=LowAFRatioToBackground,Description="old">',)))
    assert T.output_lines(declared, "LowAFRatioToBackground", "new") == declared.edited_lines(with_model=False,
                                                                                               with_blacklist=False)
    with pytest.raises(NotImplementedError):
        T.afr_params(VcfHeader(D.header(1, bg="Number=A,Type=String")), 10, 0, 0, "X")


def test_cli_parsing():
    from variantcalling_b200 import low_af_ratio as T

    a = T.parse_args(["in.vcf.gz", "out.vcf.gz"])
    assert (a.af_ratio_threshold, a.af_ratio_threshold_h_indels, a.tumor_vaf_threshold_h_indels, a.new_filter) == \
        (10, 0, 0, "LowAFRatioToBackground")
    a = T.parse_args(["i", "o", "--af_ratio_threshold", "3", "--af_ratio_threshold_h_indels", "2",
                      "--tumor_vaf_threshold_h_indels", "0.15", "--new_filter", "X"])
    assert (a.af_ratio_threshold, a.af_ratio_threshold_h_indels, a.tumor_vaf_threshold_h_indels, a.new_filter) == \
        (3.0, 2.0, 0.15, "X")
    assert T.filter_description(a.af_ratio_threshold, a.af_ratio_threshold_h_indels, a.tumor_vaf_threshold_h_indels).endswith(
        "For snps and non-h-indels: 3.0, and for h-indels (applied only if tumor VAF<0.15: 2.0)")
    for bad in ("A;B", "PASS", "RefCall", "a b", "x=y", "", "Z" * 64):
        with pytest.raises(ValueError):
            T.check_filter_id(bad)
    from ugvc.__main__ import TOOLS

    assert TOOLS["filter_low_af_ratio_to_background"] == "variantcalling_b200.low_af_ratio"
