"""GPU: the device file path (ugvc_filter_bgzf_edits) for every flag but --treat_multiallelics -- blacklists, model-less
runs, --recalibrate_genotype, INFO/END in the index -- writes the same text and index as the host writer (--host_io)
and as the oracle, and the ranges it hands back still come out equal."""
import ctypes as C
import gzip
import logging
import pickle

import numpy as np
import pytest

from oracle import ref_pipeline as R
from oracle import tabix_ref
from oracle.vcf_reader import OracleVariantFile
from tests import util
from variantcalling_b200 import bgzf_io, lib
from variantcalling_b200 import filter_variants_pipeline as fvp
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader

pytestmark = pytest.mark.gpu

END_HDR = '##INFO=<ID=END,Number=1,Type=Integer,Description="End position of the variant">'
XEND_HDR = '##INFO=<ID=XEND,Number=1,Type=Integer,Description="Not END">'


class Blacklist:  # the attribute contract of ugbio_filtering.blacklist.Blacklist
    def __init__(self, blacklist, annotation):
        self.blacklist, self.annotation, self.description = blacklist, annotation, ""
        self.selection_fcn = None  # VariantSelectionFunctions.ALL


FILTERS = [".", "PASS", "LowQual", "PASS;LowQual"]


def _edit(lines, with_end=False):
    """Input FILTER ., PASS, LowQual and PASS;LowQual; CG insertions / deletions; phased GTs; and with_end INFO/END
    pieces: long ENDs first and last, END=1 (not beyond POS), XEND= (not the key), symbolic <DEL> / <DUP> records."""
    out = []
    for i, line in enumerate(lines):
        c = line.split("\t")
        c[6] = FILTERS[i % 4]
        if i % 11 == 3:
            c[3], c[4] = "C", "CCG"
        elif i % 11 == 7:
            c[3], c[4] = "GGC", "G"
        if i % 5 == 2 and len(c) > 9:
            c[9] = c[9].replace("/", "|", 1)
        if with_end:
            pos = int(c[1])
            k = i % 6
            if k == 1:
                c[7] = f"END={pos + 25000};" + c[7]
            elif k == 2:
                c[7] = c[7] + f";END={pos + 700}"
            elif k == 3:
                c[7] = c[7] + ";END=1"
            elif k == 4:
                c[7] = f"XEND={pos + 90000};" + c[7]
            elif k == 5:  # the CNV flavour's symbolic records: the interval is the deletion / duplication
                c[3], c[4] = c[3][0], "<DEL>" if i % 12 == 5 else "<DUP>"
                c[7] = f"END={pos + 50000};" + c[7]
        out.append("\t".join(c))
    return out


@pytest.fixture(scope="module")
def job(tmp_path_factory):
    d = tmp_path_factory.mktemp("fileflags")
    ds = util.make_dataset(n_records=6000, n_custom=4, seed=17, region=("chr1", 1, 3_000_000))
    extra = util.make_dataset(n_records=600, n_custom=4, seed=18, contigs={"chr2": 242193529, "chr3": 198295559})
    lines = _edit(ds["lines"] + extra["lines"])
    header = ds["header"]
    vf = OracleVariantFile(("\n".join(header) + "\n" + "\n".join(lines) + "\n").encode())
    ds2 = dict(ds, lines=lines, vf=vf, labels=np.concatenate((ds["labels"], extra["labels"])))
    _, tr, x = util.fit_transformer(ds2)
    model = util.fit_model("gb_small", x, ds2["labels"])
    vcf = str(d / "in.vcf.gz")
    bgzf_io.write_vcf_gz(vcf, header, lines)
    mpath = str(d / "model.pkl")
    with open(mpath, "wb") as fh:
        pickle.dump({"transformer": tr, "xgb": model}, fh)
    y3 = np.where(x[:, 2] > 0, 2, ds2["labels"])
    model3 = util.fit_model("gb3", x, y3)
    m3path = str(d / "model3.pkl")
    with open(m3path, "wb") as fh:
        pickle.dump({"transformer": tr, "xgb": model3}, fh)
    chr1 = [int(l.split("\t")[1]) for l in lines if l.startswith("chr1\t")]
    cg = [int(l.split("\t")[1]) for i, l in enumerate(lines) if i % 11 in (3, 7) and l.startswith("chr1\t")]
    # overlapping blacklists, one with positions on other contigs only, one empty; hits that are CG records too
    bls = [Blacklist({("chr1", p) for p in chr1[::37]} | {("chr1", p) for p in cg[:20]} | {("chr2", 5)}, "ILLUMINA_FP"),
           Blacklist({("chr1", p) for p in chr1[::74]} | {("chr3", 7)}, "COHORT_FP"),
           Blacklist({("chr9", 1), ("chrX", 2)}, "ELSEWHERE"),
           Blacklist(set(), "EMPTY")]
    blpath = str(d / "bl.pkl")
    with open(blpath, "wb") as fh:
        pickle.dump(bls, fh)
    return dict(dir=d, vcf=vcf, header=header, lines=lines, vf=vf, customs=ds["customs"], tr=tr, model=model, mpath=mpath,
                model3=model3, m3path=m3path, bls=bls, blpath=blpath)


def _records(path):
    return [l for l in gzip.open(path).read().decode().split("\n")[:-1] if not l.startswith("#")]


def _run_both(job, name, argv, caplog):
    """The CLI on the default path and with --host_io; the default run must have stayed on the device."""
    outs = []
    totals = []
    for host in (False, True):
        out = str(job["dir"] / f"{name}{'_host' if host else ''}.vcf.gz")
        caplog.clear()
        with caplog.at_level(logging.INFO):
            totals.append(fvp.run(argv + ["--output_file", out] + (["--host_io"] if host else [])))
        text = caplog.text
        if not host:
            assert "device file path, ms on the GPU" in text and "taking the host path" not in text, "not on the device path"
        outs.append(out)
    assert gzip.open(outs[0]).read() == gzip.open(outs[1]).read(), "device and --host_io texts differ"
    assert totals[0] == totals[1]
    return outs, totals[0]


def _customs(job):
    return [a for c in job["customs"] for a in ("--custom_annotations", c)]


def test_model_cg_and_blacklists(job, caplog):
    argv = ["--input_file", job["vcf"], "--model_file", job["mpath"], "--blacklist", job["blpath"],
            "--blacklist_cg_insertions"] + _customs(job)
    (dev, _), totals = _run_both(job, "model_bl", argv, caplog)
    exp = R.filter_variants(job["vf"], job["model"], job["tr"], custom_annotations=job["customs"], blacklist_cg=True,
                            position_blacklists=[(b.blacklist, b.annotation) for b in job["bls"]])
    recs = _records(dev)
    assert recs == exp["lines"]
    both = [r for r in recs if "BLACKLST=CG_NON_HMER_INDEL,ILLUMINA_FP" in r]
    assert both and any("ILLUMINA_FP,COHORT_FP" in r for r in recs)
    assert totals["n_blacklisted"] == sum("BLACKLST=" in r for r in recs)


@pytest.mark.parametrize("flags", [["--blacklist_cg_insertions"], ["--blacklist", "BL"], ["--blacklist", "BL", "--blacklist_cg_insertions"]],
                         ids=["cg_only", "blacklist_only", "both"])
def test_model_less(job, caplog, flags):
    name = "noml_" + "_".join(f.strip("-")[:4] for f in flags)
    flags = [job["blpath"] if f == "BL" else f for f in flags]
    argv = ["--input_file", job["vcf"]] + flags
    (dev, _), totals = _run_both(job, name, argv, caplog)
    with_bl = "--blacklist" in flags
    exp = R.filter_variants(job["vf"], None, None, blacklist_cg="--blacklist_cg_insertions" in flags,
                            position_blacklists=[(b.blacklist, b.annotation) for b in job["bls"]] if with_bl else None)
    recs = _records(dev)
    assert recs == exp["lines"]
    assert not any("TREE_SCORE" in r for r in recs)
    assert {r.split("\t")[6] for r in recs} == {"PASS", "LowQual", "PASS;LowQual"}  # "." -> PASS, the rest as it is
    assert totals["n_blacklisted"] == sum("BLACKLST=" in r for r in recs) > 0
    if "--blacklist_cg_insertions" in flags:
        assert sum("CG_NON_HMER_INDEL" in r for r in recs) == totals["n_cg"] > 0


@pytest.mark.parametrize("owq", [False, True], ids=["gq", "gq_qual"])
def test_recalibrate_genotype(job, caplog, owq):
    argv = ["--input_file", job["vcf"], "--model_file", job["m3path"], "--recalibrate_genotype"] + \
        (["--overwrite_qual_tag"] if owq else []) + _customs(job)
    (dev, _), _ = _run_both(job, f"recal{int(owq)}", argv, caplog)
    exp = R.filter_variants(job["vf"], job["model3"], job["tr"], custom_annotations=job["customs"], recalibrate_genotype=True,
                            overwrite_qual_tag=owq)
    recs = _records(dev)
    bad = [i for i, (a, b) in enumerate(zip(recs, exp["lines"])) if a != b]
    # as in test_gpu_cli: int() of a phred on an integer boundary may differ in the last ulp of log10 (~1 in 10^5)
    assert len(recs) == len(exp["lines"]) and len(bad) <= 1, recs[bad[0]] if bad else None
    assert any("|" in r.split("\t")[9].split(":")[0] for r in recs)
    assert not any("TREE_SCORE" in r for r in recs)


def test_info_end_in_the_index(job, caplog):
    """A header with INFO/END: the device path ends index intervals at END beyond POS, like the host writer, so that
    queries that overlap only the tail of a long record find it."""
    header = list(job["header"])
    header.insert(len(header) - 1, END_HDR)
    header.insert(len(header) - 1, XEND_HDR)
    lines = _edit(job["lines"], with_end=True)
    vcf = str(job["dir"] / "in_end.vcf.gz")
    bgzf_io.write_vcf_gz(vcf, header, lines)
    (dev, host), _ = _run_both(job, "end", ["--input_file", vcf, "--blacklist_cg_insertions"], caplog)
    vf = OracleVariantFile(("\n".join(header) + "\n" + "\n".join(lines) + "\n").encode())
    assert _records(dev) == R.filter_variants(vf, None, None, blacklist_cg=True)["lines"]
    idx_d, idx_h = tabix_ref.TabixIndex(dev + ".tbi"), tabix_ref.TabixIndex(host + ".tbi")
    long_recs = [l.split("\t") for l in lines if l.startswith("chr1\t") and ";END=" in ";" + l.split("\t")[7]]
    tails = [(int(c[1]) + 20000, int(c[1]) + 20001) for c in long_recs if f"END={int(c[1]) + 25000}" in c[7]][:5]
    tails += [(int(c[1]) + 45000, int(c[1]) + 45001) for c in long_recs if c[4] in ("<DEL>", "<DUP>")][:5]
    assert len(tails) == 10
    for beg, end in tails + [(0, 5000), (1_000_000, 1_040_000), (2_990_000, 3_100_000)]:
        got_d = tabix_ref.query(dev, idx_d, "chr1", beg, end)
        assert got_d == tabix_ref.query(host, idx_h, "chr1", beg, end)
        if (beg, end) in tails:
            assert got_d, (beg, end)  # only the END interval reaches here


def test_out_end_and_text_equal_the_host_rules(gpu_ctx):
    """The writer on caller bytes: out_end equals ugvc_info_end on crafted INFO columns, and the text equals
    ugvc_splice_records with the same blacklist code (model-less plan)."""
    ds = util.make_dataset(n_records=400, n_custom=0, seed=23)
    infos = ["END=5000", "A=1;END=77", "END=", "END=12a", "END=12345678901", "END=1234567890", "XEND=9;END=4", "END=3;END=9",
             "ENDX=4", "A=END=5", "END=0", "END=-4", "END=7;X", "Y;END=000123"]
    lines = []
    for i, l in enumerate(ds["lines"]):
        c = l.split("\t")
        c[7] = infos[i % len(infos)] if i % 3 else c[7]
        if i % 7 == 0:
            c[3], c[4] = c[3][0], "<DEL>"
        lines.append("\t".join(c))
    text = ("\n".join(lines) + "\n").encode()
    gpu_ctx.load_plan(MC.compile_plan_no_model(VcfHeader(ds["header_text"])).blob)
    gpu_ctx.reserve(len(text) + (1 << 20), len(lines) + 64, 1)
    res = gpu_ctx.filter_batch(text, 30.0)
    n = res["n_records"]
    buf = np.frombuffer(text, dtype=np.uint8)
    want_end = fvp.info_end_positions(buf, res["line_start"], res["recinfo"], n)
    pos = np.sort(res["recinfo"]["pos"][::5].astype(np.int64))
    bl = [("A;PASS;B", pos), ("PASS", pos[::2]), ("C", np.zeros(0, np.int64))]
    comp = np.frombuffer(bgzf_io.compress_bytes(text), dtype=np.uint8)
    got = gpu_ctx.filter_bgzf_edits(comp, 0, len(text), 30.0, lib.FILE_BLACKLIST_CG, n + 64, with_model=False, blacklists=bl,
                                    want_end=True)
    assert got is not None and got["n_records"] == n
    assert np.array_equal(got["end"], want_end) and (want_end > 0).sum() > 50
    # the host writer with the code of blacklist_codes: CG first, then the blacklists in order
    code = (res["recinfo"]["flags"] & 1).astype(np.int32)
    parts = ["CG_NON_HMER_INDEL"] + [a for a, _ in bl]
    for k, (_a, p) in enumerate(bl):
        code += np.isin(res["recinfo"]["pos"].astype(np.int64), p).astype(np.int32) << (k + 1)
    strings = [";".join(parts[k] if (c >> k) & 1 else "PASS" for k in range(len(parts))).encode() for c in range(1 << len(parts))]
    table = np.frombuffer(b"".join(strings), dtype=np.uint8)
    off = np.concatenate(([0], np.cumsum([len(x) for x in strings]))).astype(np.int64)
    out = np.empty(buf.size + n * 128 + 1024, dtype=np.uint8)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    nb = lib.load_library().ugvc_splice_records(p(buf), p(res["line_start"]), p(res["recinfo"]), None, None, n, 0, 0, p(code),
                                                p(table), p(off), None, 0, p(out), out.size, None, 2)
    assert nb > 0 and gzip.decompress(got["bgzf"].tobytes()) == out[:nb].tobytes()
    assert got["n_blacklisted"] == int(np.count_nonzero(code)) > 0


def test_handed_back_ranges_are_still_equal(job, caplog):
    """A model-less run over a file with an INFO that already holds BLACKLST= and one that is ".": the device writer hands
    that range back (UGVC_E_FALLBACK) and the host writer writes it; the file equals --host_io."""
    lines = list(job["lines"])
    c = lines[10].split("\t")
    c[7] = "BLACKLST=OLD;" + c[7]
    lines[10] = "\t".join(c)
    c = lines[20].split("\t")
    c[7] = "."
    lines[20] = "\t".join(c)
    vcf = str(job["dir"] / "in_back.vcf.gz")
    bgzf_io.write_vcf_gz(vcf, job["header"], lines)
    outs = []
    for host in (False, True):
        out = str(job["dir"] / f"back{int(host)}.vcf.gz")
        caplog.clear()
        with caplog.at_level(logging.INFO):
            fvp.run(["--input_file", vcf, "--blacklist_cg_insertions", "--output_file", out] + (["--host_io"] if host else []))
        if not host:
            assert "taking the host path" in caplog.text
        outs.append(out)
    assert gzip.open(outs[0]).read() == gzip.open(outs[1]).read()


# FORMAT / sample shapes of --recalibrate_genotype (hostio.cpp recalibrated_sample): the first GQ / PL / GT key gets the
# new value, missing keys are appended in the order GQ, PL, GT, values are padded with "." (and cut to the keys),
# FORMAT "." has no keys, the other samples stay as they are
SAMPLE_SHAPES = [
    None,                                        # GT:AD:DP:GQ:PL as generated
    (".", "."),                                  # FORMAT "."
    ("GT:DP", "0|1:12"),                         # phased, GQ and PL missing
    ("AD", "3,4"),                               # GQ, PL and GT missing
    ("GT:AD:DP:GQ:PL", "0/1:3,4"),               # fewer values than keys
    ("GT:GT:DP", "0/1:1|1:5"),                   # GT twice: the first is set, the second's '|' still decides
    ("DP:GQ", "7:9:11:13"),                      # more values than keys
    ("GT:DP", None),                             # FORMAT without a sample column
    ("", None),                                  # no FORMAT column at all
]


def _recal_lines(lines):
    out = []
    for i, line in enumerate(lines):
        c = line.split("\t")
        shape = SAMPLE_SHAPES[i % len(SAMPLE_SHAPES)]
        if shape is not None:
            fmt, smp = shape
            c = c[:8] + ([fmt] if fmt else []) + ([smp] if smp is not None else [])
        if i % 4 == 1 and len(c) > 9:
            c.append("1/1:1,2:3:4:5,6,7")            # a second sample, copied as it is
        alt = c[4].split(",")[0]
        c[4] = {0: ".", 1: alt, 2: alt + ("," + ("T" if "T" not in c[3] + alt else "G"))}[(i // 3) % 3]  # 1, 2, 3 alleles
        out.append("\t".join(c))
    return out


def _recal_phreds(n, n_classes, rng):
    ph = rng.uniform(0.0, 80.0, size=(n, n_classes))
    ph[::5] = 17.25                                  # every phred ties: GQ 0, the first genotype
    ph[1::5, :2] = [[5.2, 5.9]]                      # PLs tie at 5 (the doubles do not): the first of them
    ph[2::5, 1:] = ph[2::5, :1]                      # the minimum is shared from the first column on
    return ph


def _host_writer(buf, res, low, qual, phreds, owq):
    n = res["n_records"]
    out = np.empty(buf.size + n * 256 + 4096, dtype=np.uint8)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    nb = lib.load_library().ugvc_splice_records(p(buf), p(res["line_start"]), p(res["recinfo"]), p(low), p(qual), n, int(owq), 1,
                                                None, None, None, p(phreds), phreds.shape[1], p(out), out.size, None, 2)
    assert nb > 0
    return out[:nb].tobytes()


@pytest.mark.parametrize("n_classes", [3, 6])
@pytest.mark.parametrize("owq", [False, True], ids=["gq", "gq_qual"])
def test_recalibrated_samples_equal_the_host_writer(gpu_ctx, n_classes, owq):
    """The device writer on every FORMAT / sample shape, 1, 2 and 3 alleles (n_pl = 1, 3, or capped at n_classes) and
    tied phreds, with the records' recinfo from K1 and the phreds given: the same text as ugvc_splice_records."""
    ds = util.make_dataset(n_records=900, n_custom=0, seed=29)
    text = ("\n".join(_recal_lines(ds["lines"])) + "\n").encode()
    gpu_ctx.load_plan(MC.compile_plan_no_model(VcfHeader(ds["header_text"])).blob)
    gpu_ctx.reserve(len(text) + (1 << 20), 2048, 1)
    res = gpu_ctx.filter_batch(text, 30.0)
    n = res["n_records"]
    assert n == 900
    na = (res["recinfo"]["flags"] >> 1) & 0x7F
    assert {1, 2, 3} <= set(na.tolist())
    rng = np.random.default_rng(n_classes)
    phreds = _recal_phreds(n, n_classes, rng)
    low = (rng.uniform(size=n) < 0.5).astype(np.uint8)
    qual = rng.uniform(0.0, 60.0, size=n)
    buf = np.frombuffer(text, dtype=np.uint8)
    got = gpu_ctx.test_write_records(buf, res["line_start"], res["recinfo"], lib.FILE_OVERWRITE_QUAL if owq else 0, low_score=low,
                                     qual=qual, phreds=phreds, recalibrate_genotype=True)
    assert got is not None, "clean records handed back"
    want = _host_writer(buf, res, low, qual, phreds, owq)
    if got["text"] != want:
        a, b = got["text"].split(b"\n"), want.split(b"\n")
        k = next(i for i in range(len(b)) if a[i] != b[i])
        raise AssertionError(f"record {k}: {a[k]!r} != {b[k]!r}")
    assert b"GQ:PL:GT\t" in want and b"|" in want and b"\t1/1:1,2:3:4:5,6,7" in want


# phreds the device writer hands back (UGVC_E_FALLBACK): the host writer's int() casts would not be exact, or --overwrite_qual_tag
# would print GQ in exponent form
BAD_PHREDS = {"nan": ([1.0, np.nan, 9.0], False), "inf": ([1.0, np.inf, 9.0], False),
              "beyond int32": ([1.0, 3.0e9, 9.0], False), "exponent GQ": ([0.5, 2.0e6, 3.0e6], True)}


@pytest.mark.parametrize("case", list(BAD_PHREDS) + ["one class"])
def test_recalibration_hand_backs(gpu_ctx, case):
    ds = util.make_dataset(n_records=200, n_custom=0, seed=31)
    text = ("\n".join(ds["lines"]) + "\n").encode()
    gpu_ctx.load_plan(MC.compile_plan_no_model(VcfHeader(ds["header_text"])).blob)
    gpu_ctx.reserve(len(text) + (1 << 20), 512, 1)
    res = gpu_ctx.filter_batch(text, 30.0)
    n = res["n_records"]
    rng = np.random.default_rng(5)
    phreds = rng.uniform(0.0, 80.0, size=(n, 1 if case == "one class" else 3))
    low, qual = np.zeros(n, np.uint8), rng.uniform(0.0, 60.0, size=n)
    buf = np.frombuffer(text, dtype=np.uint8)
    owq = False
    if case != "one class":
        row, owq = BAD_PHREDS[case]
        phreds[117] = row
    flags = lib.FILE_OVERWRITE_QUAL if owq else 0
    kw = dict(low_score=low, qual=qual, recalibrate_genotype=True)
    assert gpu_ctx.test_write_records(buf, res["line_start"], res["recinfo"], flags, phreds=phreds, **kw) is None, case
    if case == "exponent GQ":  # the same phreds without the QUAL overwrite stay on the device, and agree
        got = gpu_ctx.test_write_records(buf, res["line_start"], res["recinfo"], 0, phreds=phreds, **kw)
        assert got is not None and got["text"] == _host_writer(buf, res, low, qual, phreds, False)
    if case != "one class":  # the clean phreds go through
        phreds[117] = [1.5, 20.0, 30.0]
        got = gpu_ctx.test_write_records(buf, res["line_start"], res["recinfo"], flags, phreds=phreds, **kw)
        assert got is not None and got["text"] == _host_writer(buf, res, low, qual, phreds, owq)


def test_outgrown_text_buffer_hands_back(gpu_ctx):
    """Annotations long enough to outgrow the writer's text buffer hand the range back instead of failing the call."""
    ds = util.make_dataset(n_records=300, n_custom=0, seed=37)
    text = ("\n".join(ds["lines"]) + "\n").encode()
    gpu_ctx.load_plan(MC.compile_plan_no_model(VcfHeader(ds["header_text"])).blob)
    gpu_ctx.reserve(len(text) + 4096, 512, 1)
    comp = np.frombuffer(bgzf_io.compress_bytes(text), dtype=np.uint8)
    pos = np.sort(gpu_ctx.filter_batch(text, 30.0)["recinfo"]["pos"].astype(np.int64))
    bl = [("X" * 120 + str(k), pos) for k in range(30)]  # ~3.7 KiB of BLACKLST on every record
    assert gpu_ctx.filter_bgzf_edits(comp, 0, len(text), 30.0, 0, 512, with_model=False, blacklists=bl) is None
    got = gpu_ctx.filter_bgzf_edits(comp, 0, len(text), 30.0, 0, 512, with_model=False, blacklists=[("SHORT", pos)])
    assert got is not None and got["n_blacklisted"] == 300
