"""``python ugvc evaluate_concordance`` -- precision / recall of a compared call set
(``ugvc/pipelines/evaluate_concordance.py:31-108`` of the reference: same flags, same outputs).

The comparison frame comes from ``run_comparison_pipeline`` (``rtg vcfeval`` + annotation, out of
scope here).  The reference stores it as HDF5, which needs PyTables; this tool reads ``.h5`` when
PyTables is importable and also accepts ``.parquet`` / ``.csv`` exports of the same frame.  The
metrics come from ``variantcalling_b200.concordance`` (CUDA, no CPU path):
    <prefix>.stats.csv       calc_accuracy_metrics, ';'-separated (:100-101)
    <prefix>.thresholds.csv  group, threshold of calc_recall_precision_curve (:103-107)
    <prefix>.h5              both frames, when PyTables is available
"""
from __future__ import annotations

import argparse
import logging
import sys

import pandas as pd

from variantcalling_b200 import concordance

logger = logging.getLogger(__name__)


def parse_args(argv: list[str]):
    ap_var = argparse.ArgumentParser(prog="evaluate_concordance.py", description=run.__doc__)
    ap_var.add_argument("--input_file", help="Name of the input h5 file", type=str, required=True)
    ap_var.add_argument("--output_prefix", help="Prefix to output files", type=str, required=True)
    ap_var.add_argument("--dataset_key", help="h5 dataset name, such as chromosome name", default="all")
    ap_var.add_argument("--score_key", help="info key name for calculating the score", default="tree_score")
    ap_var.add_argument("--ignore_genotype", help="ignore genotype when comparing to ground-truth", action="store_true",
                        default=False)
    ap_var.add_argument("--ignore_filters", help="comma separated list of filters to ignore", default="HPOL_RUN")
    ap_var.add_argument("--output_bed", help="output bed files of fp/fn/tp per variant-type", action="store_true",
                        default=False)
    ap_var.add_argument("--use_for_group_testing", help="Column in the h5 to use for grouping (or generate default groupings)",
                        type=str)
    ap_var.add_argument("--verbosity", help="Verbosity: ERROR, WARNING, INFO, DEBUG", required=False, default="INFO")
    ap_var.add_argument("--device", help="CUDA device ordinal", type=int, default=0)
    return ap_var.parse_args(argv)


def read_frame(path: str, key: str) -> pd.DataFrame:
    low = path.lower()
    if low.endswith(".parquet"):
        return pd.read_parquet(path)
    if low.endswith((".csv", ".csv.gz", ".tsv", ".tsv.gz")):
        return pd.read_csv(path, sep="\t" if ".tsv" in low else ",")
    try:
        import tables  # noqa: F401
    except ImportError as err:
        raise ImportError("reading the comparison HDF5 needs PyTables; export the frame as .parquet or .csv") from err
    if key != "all":
        return pd.read_hdf(path, key=key)
    skip = {"concordance", "scored_concordance", "input_args", "comparison_result"}  # :80-83
    with pd.HDFStore(path, mode="r") as store:
        keys = [k.lstrip("/") for k in store.keys() if k.lstrip("/") not in skip]
        return pd.concat([store[k] for k in keys])


def run(argv: list[str]):
    """Calculate precision and recall for compared HDF5"""
    args = parse_args(argv)
    logging.basicConfig(format="%(asctime)s %(message)s", level=getattr(logging, args.verbosity))
    if args.output_bed:
        raise NotImplementedError("--output_bed (BED files per classification) is not part of the device path")
    df = read_frame(args.input_file, args.dataset_key)
    score_column = args.score_key.lower()
    if score_column not in df.columns or all(df[score_column].isna()):
        df[score_column] = 1
        logger.warning(f"No {score_column} field in comparison hdf input, expect invalid recall/precision curves")
    df["tree_score"] = df[score_column]
    classify_column = "classify" if args.ignore_genotype else "classify_gt"
    ignored_filters = args.ignore_filters.split(",")
    ctx = concordance.ConcordanceContext(args.device)
    accuracy_df = concordance.calc_accuracy_metrics(df, classify_column, ignored_filters, args.use_for_group_testing, ctx=ctx)
    accuracy_df.to_csv(f"{args.output_prefix}.stats.csv", sep=";", index=False)
    curve_df = concordance.calc_recall_precision_curve(df, classify_column, ignored_filters, args.use_for_group_testing,
                                                       ctx=ctx)
    curve_df[["group", "threshold"]].to_csv(f"{args.output_prefix}.thresholds.csv", index=None)
    try:
        import tables  # noqa: F401

        accuracy_df.to_hdf(f"{args.output_prefix}.h5", key="optimal_recall_precision")
        curve_df.to_hdf(f"{args.output_prefix}.h5", key="recall_precision_curve")
    except ImportError:
        logger.warning("PyTables is not installed: %s.h5 not written (the .csv outputs are complete)", args.output_prefix)
    ctx.close()
    return accuracy_df, curve_df


def main():
    run(sys.argv[1:])


if __name__ == "__main__":
    main()
