"""GPU: --treat_multiallelics on the device file path (ugvc_filter_bgzf_split: inflate, index pass, split build, scored
pass, merge, score math, record writer and deflate chained on the device) writes the same text and index as the host
route (--host_io: NumPy score math, host splicer) and as the oracle, raises what the host route raises, hands single
contigs back, and its score kernel (ma_score) agrees with multiallelics.score_math."""
import gzip
import logging
import pickle

import numpy as np
import pandas as pd
import pytest

from oracle import ref_pipeline as R
from oracle import tabix_ref
from oracle.vcf_reader import OracleVariantFile
from tests import multiallelic_data as MD
from tests import util
from tests.test_gpu_y_fileflags import Blacklist
from variantcalling_b200 import bgzf_io, multiallelics
from variantcalling_b200 import filter_variants_pipeline as fvp

pytestmark = pytest.mark.gpu

DEVICE_LINE = "device split path, ms on the GPU"
HANDED_BACK = "taking the host path"
END_HDR = '##INFO=<ID=END,Number=1,Type=Integer,Description="End position of the variant">'
GP_HDR = '##FORMAT=<ID=GP,Number=G,Type=Float,Description="Genotype probabilities">'


def _three_contigs(ds):
    """The case's two contigs and a third, chrM3: chrM2's records and sequence again (three contigs, so that contigs begin
    and end inside BGZF blocks)."""
    ds = dict(ds)
    ds["ref"] = dict(ds["ref"], chrM3=ds["ref"]["chrM2"])
    extra = ["chrM3\t" + ln.split("\t", 1)[1] for ln in ds["lines"] if ln.startswith("chrM2\t")]
    ds["lines"] = list(ds["lines"]) + extra
    at = next(i for i, h in enumerate(ds["header"]) if h.startswith("##contig=<ID=chrM2"))
    ds["header"] = ds["header"][:at + 1] + [ds["header"][at].replace("chrM2", "chrM3")] + ds["header"][at + 1:]
    return ds


def _vf(header, lines):
    return OracleVariantFile(("\n".join(header) + "\n" + "\n".join(lines) + "\n").encode())


_JOBS = {}


def _job(tmp_path_factory, kind):
    """The three-contig case with a `kind` model, its FASTA, model pickle and blacklists (made once per kind)."""
    if kind not in _JOBS:
        _JOBS[kind] = _make_job(tmp_path_factory, kind)
    return _JOBS[kind]


@pytest.fixture(scope="module", params=["rf", "lr", "gb3"])
def job(request, tmp_path_factory):
    return _job(tmp_path_factory, request.param)


@pytest.fixture(scope="module")
def rf_job(tmp_path_factory):
    return _job(tmp_path_factory, "rf")


@pytest.fixture(scope="module")
def gb3_job(tmp_path_factory):
    return _job(tmp_path_factory, "gb3")


def _make_job(tmp_path_factory, kind):
    d = tmp_path_factory.mktemp("filesplit_" + kind)
    ds, tr, model, split = util.make_multiallelic_case(21, kind)
    ds = _three_contigs(ds)
    fasta = str(d / "ref.fa")
    with open(fasta, "w") as fh:
        fh.write(MD.fasta_text(ds["ref"]))
    mpath = str(d / "model.pkl")
    with open(mpath, "wb") as fh:
        pickle.dump({"transformer": tr, "xgb": model}, fh)
    # blacklists with positions on merged (multi-allelic) records and on plain ones
    multi = [(ln.split("\t")[0], int(ln.split("\t")[1])) for ln in ds["lines"] if "," in ln.split("\t")[4]]
    plain = [(ln.split("\t")[0], int(ln.split("\t")[1])) for ln in ds["lines"] if "," not in ln.split("\t")[4]]
    bls = [Blacklist(set(multi[::3]) | set(plain[::29]), "ILLUMINA_FP"), Blacklist(set(multi[::7]), "COHORT_FP")]
    blpath = str(d / "bl.pkl")
    with open(blpath, "wb") as fh:
        pickle.dump(bls, fh)
    return dict(dir=d, ds=ds, tr=tr, model=model, mpath=mpath, fasta=fasta, bls=bls, blpath=blpath, split=split)


def _write(job, name, header, lines):
    vcf = str(job["dir"] / f"{name}.vcf.gz")
    bgzf_io.write_vcf_gz(vcf, header, lines)
    return vcf


def _argv(job, vcf, *extra, mpath=None):
    argv = ["--input_file", vcf, "--model_file", mpath or job["mpath"], "--treat_multiallelics", "--ref_fasta", job["fasta"], *extra]
    for c in job["ds"]["customs"]:
        argv += ["--custom_annotations", c]
    return argv


def _index_in_text_offsets(path):
    """The .tbi of `path` with every virtual offset turned into an offset of the uncompressed file: two files that hold
    the same text in differently compressed blocks have equal such indexes exactly when their .tbi say the same."""
    blocks = tabix_ref.read_bgzf_blocks(path)
    ustart = dict(zip([b[0] for b in blocks], np.concatenate(([0], np.cumsum([b[2] for b in blocks])))))

    def u(v):
        return int(ustart[v >> 16]) + (v & 0xFFFF)

    idx = tabix_ref.TabixIndex(path + ".tbi")
    bins = [{b: [(u(cb), u(ce)) for cb, ce in ch] for b, ch in bb.items()} for bb in idx.bins]
    return (idx.names, idx.format, idx.col_seq, idx.col_beg, idx.col_end, idx.meta, idx.skip, bins,
            [[u(v) for v in lin] for lin in idx.linear], idx.n_no_coor)


def _run_both(job, name, argv, caplog, *, device_contigs=None):
    """The CLI on the default path and with --host_io; same text, same index, same totals.  device_contigs: the contigs
    that must stay on the device (default: all, and none handed back)."""
    outs, totals = [], []
    for host in (False, True):
        out = str(job["dir"] / f"{name}{'_host' if host else ''}.vcf.gz")
        caplog.clear()
        with caplog.at_level(logging.INFO):
            totals.append(fvp.run(argv + ["--output_file", out] + (["--host_io"] if host else [])))
        text = caplog.text
        if not host:
            assert DEVICE_LINE in text, "the device split path did not run"
            if device_contigs is None:
                assert HANDED_BACK not in text, "a contig was handed back to the host path"
            log = text
        outs.append(out)
    assert gzip.open(outs[0]).read() == gzip.open(outs[1]).read(), "device and --host_io texts differ"
    assert _index_in_text_offsets(outs[0]) == _index_in_text_offsets(outs[1]), "device and --host_io indexes differ"
    assert totals[0] == totals[1]
    return outs, totals[0], log


def _records(path):
    return [ln for ln in gzip.open(path).read().decode().split("\n")[:-1] if not ln.startswith("#")]


def _compare(recs, exp):
    assert len(recs) == len(exp["lines"])
    bad = [i for i, (a, b) in enumerate(zip(recs, exp["lines"])) if a != b]
    assert not bad, f"{len(bad)} records differ, first: {recs[bad[0]]!r} vs {exp['lines'][bad[0]]!r}"


def _with_end(lines):
    """END pieces on split (multi-allelic) records and on a few plain ones."""
    out = []
    for i, ln in enumerate(lines):
        c = ln.split("\t")
        if "," in c[4] and i % 2 == 0:
            c[7] = c[7] + f";END={int(c[1]) + 300 + i}"
        elif i % 13 == 0:
            c[7] = f"END={int(c[1]) + 2000};" + c[7]
        out.append("\t".join(c))
    return out


@pytest.mark.parametrize("flags", ["plain", "recal", "blacklist", "end"])
def test_device_equals_host_io_and_the_oracle(job, caplog, flags):
    ds = job["ds"]
    header, lines = list(ds["header"]), list(ds["lines"])
    extra, kw = [], {}
    if flags == "recal":
        extra = ["--recalibrate_genotype", "--overwrite_qual_tag", "--decision_threshold", "20"]
        kw = dict(recalibrate_genotype=True, overwrite_qual_tag=True, decision_threshold=20.0)
    elif flags == "blacklist":
        extra = ["--blacklist", job["blpath"], "--blacklist_cg_insertions"]
        kw = dict(blacklist_cg=True, position_blacklists=[(b.blacklist, b.annotation) for b in job["bls"]])
    elif flags == "end":
        header.insert(len(header) - 1, END_HDR)
        lines = _with_end(lines)
    vcf = _write(job, f"in_{flags}", header, lines)
    idx = bgzf_io.read_tbi(vcf + ".tbi")
    assert len(idx) == 3 and any(vb & 0xFFFF for vb, _ve in idx.values()) and any(ve & 0xFFFF for _vb, ve in idx.values())
    (dev, _host), totals, _log = _run_both(job, flags, _argv(job, vcf, *extra), caplog)
    exp = R.filter_variants(_vf(header, lines), job["model"], job["tr"], custom_annotations=ds["customs"],
                            treat_multiallelics=True, ref_fasta=ds["ref"], **kw)
    recs = _records(dev)
    _compare(recs, exp)
    assert totals["n_records"] == len(lines)
    assert totals["n_low_score"] == sum("LOW_SCORE" in f for f in exp["filters"])
    if flags == "recal":
        n_pl = [len(r.split("\t")[9].split(":")[-1].split(",")) for r in recs]
        assert 6 in n_pl and 10 in n_pl  # noqa: PLR2004
    if flags == "blacklist":
        assert totals["n_blacklisted"] == sum("BLACKLST=" in r for r in recs) > 0
        assert any("BLACKLST=" in r and "," in r.split("\t")[4] for r in recs)  # on merged records
    if flags == "end":
        assert sum(";END=" in ";" + r.split("\t")[7] and "," in r.split("\t")[4] for r in recs) > 50  # noqa: PLR2004


def _error_of(argv):
    try:
        fvp.run(argv)
    except Exception as err:  # noqa: BLE001
        return type(err), str(err)
    return None


def _two_class_model(job):
    split = job["split"]
    with pd.option_context("future.infer_string", False):
        x = job["tr"].transform(R.harness_float_columns(split)).to_numpy(dtype=np.float64)
    y = np.array([int(any(g for g in gt if g)) for gt in split["gt"]])
    path = str(job["dir"] / "model2.pkl")
    with open(path, "wb") as fh:
        pickle.dump({"transformer": job["tr"], "xgb": util.fit_model("rf", x, y)}, fh)
    return path


@pytest.mark.parametrize("case", ["no_multiallelic", "no_cluster", "gt_assert", "number_g", "two_class"])
def test_error_contract(rf_job, case):
    job = rf_job
    ds = job["ds"]
    header, lines, mpath = list(ds["header"]), list(ds["lines"]), None
    alt = [ln.split("\t")[4] for ln in lines]
    if case == "no_multiallelic":
        lines = [ln for ln, a in zip(lines, alt) if "," not in a and "*" not in a]
    elif case == "no_cluster":
        lines = [ln for ln, a in zip(lines, alt) if "*" not in a]
    elif case in ("gt_assert", "number_g"):
        k = next(i for i, a in enumerate(alt) if a.count(",") == 1 and "*" not in a and lines[i].startswith("chrM2\t"))
        c = lines[k].split("\t")
        if case == "gt_assert":  # neither allele of the second split row is called
            c[9] = "0/0" + c[9][3:]
        else:  # a per-genotype tag other than PL on the record
            header.insert(len(header) - 1, GP_HDR)
            c[8] += ":GP"
            c[9] += ":0.1,0.2,0.3,0.1,0.2,0.1"
        lines[k] = "\t".join(c)
    else:
        mpath = _two_class_model(job)
    vcf = _write(job, f"err_{case}", header, lines)
    got = _error_of(_argv(job, vcf, mpath=mpath) + ["--output_file", str(job["dir"] / f"out_err_{case}.vcf.gz")])
    want = _error_of(_argv(job, vcf, mpath=mpath) + ["--output_file", str(job["dir"] / f"out_err_{case}_h.vcf.gz"), "--host_io"])
    expected = {"no_multiallelic": ValueError, "no_cluster": KeyError, "gt_assert": AssertionError, "number_g": RuntimeError,
                "two_class": IndexError}[case]
    assert want is not None and want[0] is expected, want
    assert got == want


def test_fallback_of_one_contig(gb3_job, caplog):
    job = gb3_job
    ds = job["ds"]
    lines = list(ds["lines"])
    k = next(i for i, ln in enumerate(lines) if ln.startswith("chrM2\t") and "," not in ln.split("\t")[4])
    c = lines[k].split("\t")
    c[7] = "TREE_SCORE=0.5;" + c[7]  # the device writer leaves such a record to the host writer
    lines[k] = "\t".join(c)
    vcf = _write(job, "in_fallback", ds["header"], lines)
    _outs, _totals, log = _run_both(job, "fallback", _argv(job, vcf), caplog, device_contigs=["chrM1", "chrM3"])
    handed = [ln for ln in log.split("\n") if HANDED_BACK in ln]
    assert len(handed) == 1 and "chrM2..chrM2" in handed[0], handed


# ---------------------------------------------------------------- the score kernel
def _ulps(a, b):
    m = np.maximum(np.abs(a), np.abs(b))
    return np.where(a == b, 0.0, np.abs(a - b) / np.spacing(np.where(m > 0, m, 1.0)))


def _gq(ph):
    s = np.sort(ph, axis=1)
    return (s[:, 1] - s[:, 0]).astype(np.int64)


def test_score_kernel_against_numpy(gpu_ctx):
    ctx = gpu_ctx
    rng = np.random.default_rng(5)
    one_minus = 1.0 - 2.0 ** -53
    report, worst = [], 0.0
    for w in (3, 6, 10, 15):
        special = [0.0, 1.0, one_minus] + [k / n for n in (3, 7, 10, 50, 100, 500) for k in range(n + 1)]
        special += [a * b for a in (0.3, 0.5, one_minus, 0.999) for b in (0.1, 0.7, 0.999, one_minus)]
        crafted = []
        for j in range(101):
            v = 10.0 ** (-j / 10) - 1e-10
            for d in range(-4, 5):
                x = v
                for _ in range(abs(d)):
                    x = np.nextafter(x, np.inf if d > 0 else -np.inf)
                crafted.append(max(0.0, x))
        vals = np.array(special + crafted)
        rows_c = np.resize(vals, ((vals.size + w - 1) // w) * w).reshape(-1, w)
        rows_c = np.concatenate((rows_c, np.roll(rows_c, 1, axis=1), np.eye(w), np.zeros((1, w))))
        rows_d = rng.dirichlet(np.ones(w), size=250_000)
        for name, rows in (("crafted", rows_c), ("dirichlet", rows_d)):
            ph, q, low = ctx.test_ma_score(rows, 30.0)
            eph, eq, elow = multiallelics.score_math(rows, 30.0)
            assert np.all(ph[rows == 0.0] == 100.0) and np.all(eph[rows == 0.0] == 100.0)  # noqa: PLR2004
            u = float(_ulps(ph, eph).max())
            worst = max(worst, u)
            n_pl = int(np.count_nonzero(ph.astype(np.int64) != eph.astype(np.int64)))
            n_gq = int(np.count_nonzero(_gq(ph) != _gq(eph)))
            # the crafted phreds lie next to integers, so many crafted quals lie within ulps of the threshold (30): ties
            tie = np.abs(eq - 30.0) <= 8 * np.spacing(30.0) if name == "crafted" else np.zeros(eq.size, bool)
            assert np.array_equal(low[~tie], elow[~tie]), (w, name)
            report.append(f"width {w} {name}: {rows.shape[0]} rows, max phred difference {u:.0f} ulp, int(PL) differs on {n_pl}, "
                          f"int(GQ) on {n_gq}, qual differs (by ulps) on {int(np.count_nonzero(q != eq))}, LOW_SCORE differs "
                          f"on {int(np.count_nonzero(low != elow))} of {int(tie.sum())} ties at the threshold")
            if name == "dirichlet":
                assert n_pl == 0 and n_gq == 0, report[-1]
        # crafted ties: the threshold is NumPy's qual of the row, so LOW_SCORE hangs on the last ulp of qual
        n_tie_diff = 0
        for r in rows_d[:40]:
            _eph, eq, elow = multiallelics.score_math(r[None, :], 0.0)
            _ph, q, low = ctx.test_ma_score(r[None, :], float(eq[0]))
            assert q[0] != eq[0] or low[0] == 1
            n_tie_diff += int(q[0] > eq[0])
        report.append(f"width {w}: {n_tie_diff} of 40 quals set as the threshold land above it on the device")
    print("\nma_score vs NumPy:\n  " + "\n  ".join(report) + f"\n  worst: {worst:.0f} ulp")
