#!/usr/bin/env python
"""Generate tests/golden/gvcf_hcr.json.gz from the REFERENCE's own gvcf_to_bed (ugvc/joint/gvcf_bed.py) and BedWriter
(ugbio_core/vcfbed/bed_writer.py).

The reference module is imported with stand-ins for pysam and tqdm: pysam.VariantFile yields duck-typed records (chrom,
start, stop, ref and samples[0] with ``in`` / ``[]``, GQ and GT typed as oracle/gvcf_hcr_ref.py types them; a literal
that cannot be typed raises while the record is read) and tqdm passes the iterable through.  Each case records the BED
text and the skipped count, or the exception type and the record it was raised at.  The corpus is the crafted records,
the error records and seeded random gVCFs of tests/gvcf_hcr_data.py, with gt True and False and thresholds 0 / 20 / 99.
Usage: python scripts/make_golden_gvcf_hcr.py /path/to/reference
"""
import gzip
import importlib.util
import json
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if len(sys.argv) != 2:  # noqa: PLR2004
    sys.exit(__doc__)
REF = sys.argv[1]  # the reference checkout's root

from oracle import gvcf_hcr_ref as R  # noqa: E402
from tests import gvcf_hcr_data as D  # noqa: E402

STATE = {"text": "", "read": 0}


class _VariantFile:
    def __init__(self, path, mode="r"):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False

    def fetch(self):
        header, data = R.records(STATE["text"])
        decl, info_end = R.gq_decl(header), "END" in header.info
        for ln in data:
            rec = R.Record(ln, decl, info_end)  # typing errors fire here, as pysam's do while reading
            STATE["read"] += 1
            yield rec


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


sys.modules["pysam"] = types.SimpleNamespace(VariantFile=_VariantFile)
tqdm_auto = types.ModuleType("tqdm.auto")
tqdm_auto.tqdm = lambda it, **kw: it
sys.modules["tqdm"] = types.ModuleType("tqdm")
sys.modules["tqdm.auto"] = tqdm_auto
for pkg in ("ugbio_core", "ugbio_core.vcfbed"):
    sys.modules[pkg] = types.ModuleType(pkg)
_load("ugbio_core.vcfbed.bed_writer", os.path.join(REF, "ugbio_utils/src/core/ugbio_core/vcfbed/bed_writer.py"))
gvcf_bed = _load("reference_gvcf_bed", os.path.join(REF, "ugvc/joint/gvcf_bed.py"))

KINDS = ((R.LiteralError, "literal"), (TypeError, "type"), (KeyError, "key"))


def run_reference(text: str, thr: int, gt: bool) -> dict:
    STATE["text"], STATE["read"] = text, 0
    with tempfile.TemporaryDirectory() as d:
        bed = os.path.join(d, "out.bed")
        try:
            skipped = gvcf_bed.gvcf_to_bed("in.g.vcf.gz", bed, thr, gt)
        except Exception as err:  # noqa: BLE001
            for cls, kind in KINDS:
                if isinstance(err, cls):
                    return {"error": [STATE["read"] - (0 if cls is R.LiteralError else 1), kind]}
            raise
        # BedWriter is never closed by gvcf_to_bed: its text is flushed when the file object goes
        import gc

        gc.collect()
        return {"bed": open(bed).read(), "skipped": skipped}


def main():
    cases = []

    def add(name, records, hdr=None):
        text = D.text(records, **(hdr or {}))
        for thr in (0, 20, 99):
            for gt in (True, False):
                cases.append({"name": name, "text": text, "gq_threshold": thr, "gt": gt,
                              "result": run_reference(text, thr, gt)})

    for name, recs in D.crafted_records():
        add(name, recs)
        add(name + "/float_gq", recs, {"gq": "Number=1,Type=Float"})
        add(name + "/no_info_end", recs, {"info_end": False})
    pre = [D.var("chr1", 100 + 10 * k, "A", "C", fmt="GT:DP", sample="0/1:5") for k in range(3)]
    for k, (rec, _kind, hdr) in enumerate(D.error_records()):
        add(f"error{k}", pre + [rec], hdr)
        add(f"error{k}/skipped", ["chr1\t400\t.\tA\t<*>\t0\t.\tEND=600\tGT:DP\t0/0:5", rec], hdr)
    for seed in range(4):
        add(f"random{seed}", D.random_records(1500, 100 + seed, overlap=1.0 + seed))
    add("alternating", D.alternating(300) + D.alternating(50, "chr2"))
    out = os.path.join(ROOT, "tests", "golden", "gvcf_hcr.json.gz")
    with gzip.open(out, "wt") as fh:
        json.dump({"source": "ugvc/joint/gvcf_bed.py:gvcf_to_bed", "cases": cases}, fh)
    print(f"{len(cases)} cases -> {out}")


if __name__ == "__main__":
    main()
