"""``python ugvc <tool> <args>`` dispatcher.

The reference routes every tool through ``ugvc/__main__.py`` (simppl
``CommandLineInterface``, ``ugvc/__main__.py:43-54,104-105``).  This repository
implements the tools of the filtering hot path -- ``filter_variants_pipeline`` and the
``evaluate_concordance`` step that scores its output against truth -- so the dispatcher knows
exactly those names and hands ``sys.argv[2:]`` to their ``run``.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TOOLS = {"filter_variants_pipeline": "variantcalling_b200.filter_variants_pipeline",
         "filter_low_af_ratio_to_background": "variantcalling_b200.low_af_ratio",
         "calibrate_bridging_snvs": "variantcalling_b200.bridging_snvs",
         "gvcf_hcr": "variantcalling_b200.gvcf_hcr",
         "evaluate_concordance": "variantcalling_b200.evaluate_concordance"}


def main(argv=None):
    argv = list(sys.argv if argv is None else argv)
    if len(argv) < 2 or argv[1] in ("-h", "--help"):  # noqa: PLR2004
        print("usage: python ugvc <tool> [args]\n\ntools:\n  " + "\n  ".join(sorted(TOOLS)))
        return 0 if len(argv) >= 2 else 1  # noqa: PLR2004
    tool = argv[1]
    if tool not in TOOLS:
        print(f"ugvc: unknown tool {tool!r}; this build provides: {', '.join(sorted(TOOLS))}", file=sys.stderr)
        return 2
    import importlib

    importlib.import_module(TOOLS[tool]).run(argv[2:])
    return 0


if __name__ == "__main__":
    sys.exit(main())
