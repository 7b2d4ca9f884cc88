"""Loading and comparing tests/golden/concordance_annotate.json.gz (written by scripts/make_golden_annotate.py from the
reference's own annotate_concordance)."""
import functools
import gzip
import json
import os

import numpy as np
import pandas as pd

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "concordance_annotate.json.gz")
_DTYPES = {"pos": np.int64, "indel": bool, "qual": np.float64}


@functools.lru_cache(maxsize=1)
def load():
    with gzip.open(GOLDEN, "rt") as fh:
        return json.load(fh)


def _cell(v):
    if v == "NaN":
        return np.nan
    return tuple(v) if isinstance(v, list) else v


def frame(fj) -> pd.DataFrame:
    """An input frame of the golden, with the dtypes the generator gave it."""
    cols = {}
    for k, c in enumerate(fj["columns"]):
        vals = [_cell(r[k]) for r in fj["rows"]]
        cols[c] = np.array(vals, dtype=_DTYPES[c]) if c in _DTYPES else pd.Series(vals, dtype=object)
    return pd.DataFrame(cols)


def write_inputs(tmp_dir) -> tuple[str, str]:
    g = load()
    fa, bed = os.path.join(tmp_dir, "ref.fa"), os.path.join(tmp_dir, "overlaps.bed")
    with open(fa, "w") as fh:
        fh.write(g["fasta"])
    with open(bed, "w") as fh:
        fh.write(g["bed"])
    return fa, bed


def genome() -> dict:
    out, name = {}, None
    for ln in load()["fasta"].splitlines():
        if ln.startswith(">"):
            name = ln[1:].split()[0]
            out[name] = []
        else:
            out[name].append(ln.strip())
    return {k: "".join(v) for k, v in out.items()}


def _py(v):
    if isinstance(v, (tuple, list, np.ndarray)):
        return [_py(x) for x in v]
    if v is None:
        return None
    if isinstance(v, (bool, np.bool_)):
        return bool(v)
    if isinstance(v, (int, np.integer)):
        return int(v)
    if isinstance(v, (float, np.floating)):
        return "NaN" if np.isnan(v) else float(v)
    return str(v)


def assert_frame_matches(got: pd.DataFrame, want: dict):
    """Cell by cell, with the column order, the dtypes and the None / NaN placement of the reference's frame."""
    assert list(got.columns) == want["columns"]
    assert [str(t) for t in got.dtypes] == want["dtypes"]
    assert len(got) == len(want["rows"])
    for k, col in enumerate(want["columns"]):
        got_col = [_py(v) for v in got[col]]
        want_col = [r[k] for r in want["rows"]]
        if got_col != want_col:
            bad = next(i for i, (a, b) in enumerate(zip(got_col, want_col)) if a != b)
            raise AssertionError(f"column {col}, row {bad}: got {got_col[bad]!r}, want {want_col[bad]!r}")


def assert_frames_equal(got: pd.DataFrame, want: pd.DataFrame):
    assert list(got.columns) == list(want.columns)
    assert [str(t) for t in got.dtypes] == [str(t) for t in want.dtypes]
    for col in want.columns:
        a, b = [_py(v) for v in got[col]], [_py(v) for v in want[col]]
        if a != b:
            bad = next(i for i, (x, y) in enumerate(zip(a, b)) if x != y)
            raise AssertionError(f"column {col}, row {bad}: got {a[bad]!r}, want {b[bad]!r}")
