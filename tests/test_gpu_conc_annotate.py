"""GPU: annotate_concordance (variantcalling_b200.concordance over csrc/conc_annotate.cu) against the reference's own
output (tests/golden/concordance_annotate.json.gz) cell by cell, its exceptions at the same records, the oracle
restatement on a million random records over a seeded genome, and the metrics of an annotated frame."""
import numpy as np
import pandas as pd
import pytest

from oracle import annotate_ref as AR
from tests import annotate_data as AD
from tests import annotate_golden as AG
from tests.test_annotate_cpu import EXCEPTIONS
from variantcalling_b200 import concordance as PC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = PC.ConcordanceContext(0)
    yield c
    c.close()


@pytest.mark.parametrize("name", sorted(AG.load()["cases"]))
def test_annotate_matches_the_reference_golden(name, ctx, tmp_path):
    case = AG.load()["cases"][name]
    fa, bed = AG.write_inputs(str(tmp_path))
    df = AG.frame(case["input"])
    before = ctx.launch_count()
    got, annots = PC.annotate_concordance(df, fa, annotate_intervals=[bed] if case["bed"] else None,
                                          flow_order=case["flow_order"], ctx=ctx)
    assert ctx.launch_count() == before + 1
    assert got is df  # annotated in place and returned, like the reference
    assert annots == case["annots"]
    AG.assert_frame_matches(got, case["output"])


@pytest.mark.parametrize("name", sorted(AG.load()["raising"]))
def test_annotate_raises_like_the_reference(name, ctx, tmp_path):
    case = AG.load()["raising"][name]
    fa, _bed = AG.write_inputs(str(tmp_path))
    with pytest.raises(EXCEPTIONS[case["exception"]]) as info:
        PC.annotate_concordance(AG.frame(case["input"]), fa, ctx=ctx)
    row = info.value.__cause__.row if info.value.__cause__ is not None else None
    assert row == case["row"] or f"record {case['row']}:" in str(info.value)


def test_contigs_stay_on_the_handle(ctx, tmp_path):
    fa, _bed = AG.write_inputs(str(tmp_path))
    df = AG.frame(AG.load()["cases"]["tgca"]["input"])
    for chrom in ("chr1", "chr2", "chr1"):  # per-contig calls, as run_comparison_pipeline makes them
        part = df[df["chrom"] == chrom].copy()
        want, _ = AR.annotate(part, AG.genome())
        got, _ = PC.annotate_concordance(part, fa, ctx=ctx)
        AG.assert_frames_equal(got, want)
    assert sum(1 for k in ctx._annot_contigs if k[0] == fa) == 2  # noqa: SLF001


def test_bigwig_coverage_is_refused(ctx, tmp_path):
    fa, _bed = AG.write_inputs(str(tmp_path))
    with pytest.raises(NotImplementedError):
        PC.annotate_concordance(AG.frame(AG.load()["cases"]["tgca"]["input"]), fa, ["hq.bw"], ["all.bw"], ctx=ctx)


def test_a_million_random_records_against_the_oracle(ctx, tmp_path):
    genome = AD.make_genome(41, {"chrA": 400_000, "chrB": 250_000, "chrC": 60_000, "chrD": 3_000})
    fa = str(tmp_path / "big.fa")
    with open(fa, "w") as fh:
        fh.write(AD.fasta_text(genome))
    df = AD.make_frame(genome, 1_000_000, 43)
    for flow in ("TGCA", "TGC"):
        want, _ = AR.annotate(df, genome, flow)
        got, _ = PC.annotate_concordance(df.copy(), fa, flow_order=flow, ctx=ctx)
        AG.assert_frames_equal(got, want)


def test_annotate_then_metrics_reproduce_the_reference(ctx, tmp_path):
    from tests.test_concordance_cpu import check_accuracy, check_curve

    m = AG.load()["metrics"]
    fa, _bed = AG.write_inputs(str(tmp_path))
    df, _ = PC.annotate_concordance(AG.frame(m["input"]), fa, ctx=ctx)
    df["tree_score"] = np.array(m["tree_score"], dtype=np.float64)
    df["classify"] = pd.Series(m["classify"], dtype=object)
    check_accuracy(PC.calc_accuracy_metrics(df.copy(), "classify", ctx=ctx), m["accuracy"])
    check_curve(PC.calc_recall_precision_curve(df.copy(), "classify", ctx=ctx), m["curve"])
