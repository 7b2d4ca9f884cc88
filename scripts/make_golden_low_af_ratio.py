#!/usr/bin/env python
"""Generate tests/golden/low_af_ratio.json.gz from the REFERENCE's own process_record
(ugbio_filtering/filter_low_af_ratio_to_background.py:75-114).

The reference module is imported with stand-ins for pysam / tqdm / the logger (import only: nothing of theirs runs), and
its process_record is called on duck-typed records whose samples are the typed values of oracle/low_af_ratio_ref.py.
Each entry is (data line, header variant, thresholds, failed or "TypeError"); the records are the crafted corpus and
seeded random multi-sample records of tests/low_af_ratio_data.py, plus the reference unit test's VCF
(tests/golden/low_af_ratio_unit.vcf).  Usage: python scripts/make_golden_low_af_ratio.py /path/to/reference/ugbio_utils/src
"""
import gzip
import importlib
import json
import logging
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if len(sys.argv) != 2:  # noqa: PLR2004
    sys.exit(__doc__)
REF = sys.argv[1]  # the reference checkout's ugbio_utils/src

for name in ("pysam", "tqdm", "tqdm.auto", "ugbio_core", "ugbio_core.logger"):
    sys.modules[name] = types.ModuleType(name)
sys.modules["tqdm"].auto = sys.modules["tqdm.auto"]
sys.modules["ugbio_core.logger"].logger = logging.getLogger("reference")
sys.path.insert(0, os.path.join(REF, "filtering"))
ref = importlib.import_module("ugbio_filtering.filter_low_af_ratio_to_background")

from oracle import low_af_ratio_ref as R  # noqa: E402
from oracle.vcf_reader import OracleHeader  # noqa: E402
from tests import low_af_ratio_data as D  # noqa: E402


class _Sample(dict):
    pass


class _Record:
    def __init__(self, samples):
        self.samples = {f"S{k}": _Sample(s) for k, s in enumerate(samples)}


HEADERS = {"A": {}, "vaf1": {"vaf": "Number=1,Type=Float"}, "bg_dot_int": {"bg": "Number=.,Type=Integer"},
           "vt_dot": {"vt": "Number=.,Type=String"}, "no_vaf": {"vaf": ""}}
THRESHOLDS = [(10, 0, 0), (10, 2, 0.15), (2, 1, 0.3), (0.05, 0.05, 1)]


def entries(text, hkey, thr):
    lines = text.split("\n")
    head = [ln for ln in lines if ln.startswith("#")]
    kinds = R.header_kinds(OracleHeader(head))
    out = []
    for ln in (ln for ln in lines if ln and not ln.startswith("#")):
        try:
            samples = R.typed_samples(ln, kinds)
        except R.LiteralError:
            continue  # refused before the rule runs
        cols = ln.split("\t")
        vt = None
        for kv in ([] if cols[7] == "." else cols[7].split(";")):
            k, sep, v = kv.partition("=")
            if k == "VARIANT_TYPE":
                vt = (v or None) if sep else None
        h = kinds["VARIANT_TYPE"] and vt == "h-indel"
        a, b = (thr[1], thr[2]) if h else (thr[0], 1)
        try:
            got = bool(ref.process_record(_Record(samples), a, b))
        except TypeError:
            got = "TypeError"
        out.append([ln, hkey, list(thr), got])
    return out


def main():
    golden = []
    for hkey, kw in HEADERS.items():
        for thr in THRESHOLDS:
            golden += entries(D.crafted_text(**kw), hkey, thr)
        golden += entries(D.random_text(3000, 4, 7, **kw), hkey, THRESHOLDS[1])
    golden += entries(D.unit_text(), "unit", THRESHOLDS[1])
    path = os.path.join(ROOT, "tests", "golden", "low_af_ratio.json.gz")
    with gzip.open(path, "wt") as fh:
        json.dump({"headers": HEADERS, "entries": golden}, fh)
    print(f"{len(golden)} entries -> {path}")


if __name__ == "__main__":
    main()
