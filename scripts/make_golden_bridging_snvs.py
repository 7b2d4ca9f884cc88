#!/usr/bin/env python
"""Generate tests/golden/bridging_snvs.json.gz from the REFERENCE's own calibrate_bridging_snvs
(ugvc/pipelines/vcfbed/calibrate_bridging_snvs.py: run, is_homopolymer_snp).

The reference module is imported with import-only stand-ins for pysam, simppl and the ugvc logger.  Its run() is then
driven, one record at a time, through a stand-in pysam whose VariantFile yields duck-typed records (sample 0's
AD / DP / BG_AD / BG_DP typed as oracle/bridging_snvs_ref.py types them, str() = the line with its newline) and whose
FastaFile slices a seeded genome (pysam's ValueError for a negative start or an unknown contig).  Each entry records the
rescue decision, the edited QUAL / FILTER, the log lines, is_homopolymer_snp's own (decision, info) or the exception
type.  The corpus is the crafted records, the error records and seeded random records of tests/bridging_snvs_data.py,
over min_query_hmer_size 0..6, min_distance_from_edge 0..2 and several thresholds; the genome is stored with it.
Usage: python scripts/make_golden_bridging_snvs.py /path/to/reference
"""
import argparse
import gzip
import importlib.util
import json
import logging
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if len(sys.argv) != 2:  # noqa: PLR2004
    sys.exit(__doc__)
REF = sys.argv[1]  # the reference checkout's root

from oracle import bridging_snvs_ref as R  # noqa: E402
from oracle.vcf_reader import OracleHeader  # noqa: E402
from tests import bridging_snvs_data as D  # noqa: E402

LOG: list[str] = []


class _Capture(logging.Handler):
    def emit(self, record):
        LOG.append(record.getMessage())


ref_logger = logging.getLogger("reference.calibrate_bridging_snvs")
ref_logger.setLevel(logging.INFO)
ref_logger.propagate = False
ref_logger.addHandler(_Capture())

STATE = {"records": [], "fasta": {}, "written": []}


class _Filter:
    def __init__(self, ids):
        self.ids = list(ids)

    def keys(self):
        return list(self.ids)

    def add(self, fid):  # htslib bcf_add_filter
        if fid in self.ids:
            return
        self.ids = [fid] if fid == "PASS" or self.ids == ["PASS"] else [*self.ids, fid]


class _Record:
    def __init__(self, line, kinds):
        cols = line.split("\t")
        self.line = line
        self.chrom, self.pos, self.ref = cols[0], int(cols[1]), cols[3]
        self.alts = None if cols[4] == "." else tuple(cols[4].split(","))
        self.qual = R.parse_qual(cols[5])
        self.filter = _Filter([] if cols[6] == "." else cols[6].split(";"))
        self.samples = [R.typed_sample0(cols, kinds)]

    def __str__(self):
        return self.line + "\n"


class _VariantFile:
    def __init__(self, path, mode="r", header=None):
        self.header = None

    def __iter__(self):
        return iter(STATE["records"])

    def write(self, record):
        STATE["written"].append(record)

    def close(self):
        pass


class _FastaFile:
    def __init__(self, path):
        pass

    def fetch(self, contig, start, end):
        if start < 0:
            raise ValueError(f"start out of range ({start})")
        if contig not in STATE["fasta"]:
            raise ValueError(f"failure when retrieving sequence on '{contig}'")
        return STATE["fasta"][contig][start:end].decode("latin-1")


def _get_parser(name, doc):
    return argparse.ArgumentParser(prog=name, description=doc)


pysam = types.ModuleType("pysam")
pysam.VariantFile, pysam.FastaFile, pysam.tabix_index = _VariantFile, _FastaFile, lambda *a, **k: None
simppl = types.ModuleType("simppl")
simppl_cli = types.ModuleType("simppl.cli")
simppl_cli.get_parser = _get_parser
simppl.cli = simppl_cli
ugvc = types.ModuleType("ugvc")
ugvc.logger = ref_logger
sys.modules.update({"pysam": pysam, "simppl": simppl, "simppl.cli": simppl_cli, "ugvc": ugvc})
spec = importlib.util.spec_from_file_location(
    "ref_calibrate_bridging_snvs", os.path.join(REF, "ugvc", "pipelines", "vcfbed", "calibrate_bridging_snvs.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

HEADERS = {"A": {}, "float": {"dp": "Number=1,Type=Float", "bg_dp": "Number=1,Type=Float", "ad": "Number=.,Type=Float"},
           "ad1": {"ad": "Number=1,Type=Integer", "bg_dp": "Number=A,Type=Integer"}, "no_bg_ad": {"bg_ad": None},
           "no_bg_dp": {"bg_dp": None}}
ARGS = [(m, 5, 0.2, 0.1, 10, d, 20) for m in range(7) for d in range(3)] + [(3, 4, 0.5, 0.0, 0, 1, 37), (5, 0, 0.2, 0.1, 10, 0, 60)]
FLAGS = ("min_query_hmer_size", "min_initial_qual", "min_tumor_vaf", "max_normal_vaf", "min_normal_depth",
         "min_distance_from_edge", "set_qual")


def entry(line, hkey, kinds, args):
    """The reference's run() on one record (a fresh stand-in VariantFile each time), and is_homopolymer_snp alone."""
    try:
        rec = _Record(line, kinds)
    except R.LiteralError:
        return None  # refused before the reference sees it (a documented deviation)
    STATE["records"], STATE["written"] = [rec], []
    LOG.clear()
    argv = ["calibrate_bridging_snvs", "--vcf", "in.vcf", "--reference", "ref.fa", "--output", "out.vcf"]
    for f, v in zip(FLAGS, args):
        argv += [f"--{f}", str(v)]
    try:
        hm = list(ref.is_homopolymer_snp(_Record(line, kinds), _FastaFile(""), args[0], args[1], args[5]))
    except Exception as err:  # noqa: BLE001
        hm = type(err).__name__
    try:
        ref.run(argv)
    except Exception as err:  # noqa: BLE001
        return [line, hkey, list(args), type(err).__name__, hm]
    out = STATE["written"][0]
    return [line, hkey, list(args), {"qual": out.qual, "filter": out.filter.keys(), "logs": list(LOG)}, hm]


def main():
    g = D.genome()
    STATE["fasta"] = g
    golden = []
    crafted = D.crafted_records(g)
    errors = [r for r, _ in D.error_records(g)]
    rnd = D.random_records(g, 2000, 5)
    for hkey, kw in HEADERS.items():
        kinds = R.header_kinds(OracleHeader(D.header(**kw).split("\n")))
        for args in ARGS if hkey == "A" else ARGS[::7]:
            for line in crafted + errors + (rnd if args[5] == 0 and args[0] in (3, 5) else []):
                e = entry(line, hkey, kinds, args)
                if e is not None:
                    golden.append(e)
    path = os.path.join(ROOT, "tests", "golden", "bridging_snvs.json.gz")
    with gzip.open(path, "wt") as fh:
        json.dump({"headers": HEADERS, "genome": {k: v.decode("latin-1") for k, v in g.items()}, "flags": FLAGS,
                   "entries": golden}, fh)
    print(f"{len(golden)} entries -> {path}")


if __name__ == "__main__":
    main()
