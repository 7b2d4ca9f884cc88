#!/usr/bin/env python
"""Format every float32 in [1e-4f, 1e6f) with the record writer's "%g" (csrc/fileio.cu: fio_format_g) on the device
and compare each with Python's "%g" (correctly rounded, round-half-even on the binary value) on host worker processes.

A value is right when the device prints exactly what "%g" prints, or hands it back (length 0) where "%g" needs the
exponent form.  Prints the number of values checked and of mismatches, with the first few mismatches; exit status 1
when there is any.  About 2.9e8 values: minutes with one worker per core.

    python scripts/check_format_g.py [--chunk 16777216] [--workers N]
"""
import argparse
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from variantcalling_b200 import lib  # noqa: E402

LO = int(np.array(1e-4, np.float32).view(np.uint32))
HI = int(np.array(1e6, np.float32).view(np.uint32))


def expected_blob(bounds) -> bytes:
    """'\\n'-terminated "%g" of every float32 with bits in [a, b), "" where "%g" uses the exponent form."""
    a, b = bounds
    v = np.arange(a, b, dtype=np.uint32).view(np.float32).astype(np.float64).tolist()
    return ("\n".join(s if "e" not in s else "" for s in ("%g" % x for x in v)) + "\n").encode()


def device_blob(out: np.ndarray) -> bytes:
    n = out[:, 15].astype(np.int64)
    slots = out.copy()
    slots[np.arange(n.size), n] = ord("\n")
    return slots[np.arange(16)[None, :] <= n[:, None]].tobytes()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--chunk", type=int, default=1 << 24)
    ap.add_argument("--workers", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args()
    ctx = lib.Context(0)
    t0 = time.time()
    checked = bad = 0
    shown = []
    pieces = 64  # host work per chunk, spread over the workers
    with ProcessPoolExecutor(a.workers) as pool:
        for c0 in range(LO, HI, a.chunk):
            c1 = min(c0 + a.chunk, HI)
            step = -(-(c1 - c0) // pieces)
            jobs = pool.map(expected_blob, [(s, min(s + step, c1)) for s in range(c0, c1, step)])
            out = ctx.test_format_g(np.arange(c0, c1, dtype=np.uint32).view(np.float32))
            got = device_blob(out)
            want = b"".join(jobs)
            checked += c1 - c0
            if got != want:
                g, w = got.split(b"\n")[:-1], want.split(b"\n")[:-1]
                idx = [i for i in range(len(w)) if g[i] != w[i]]
                bad += len(idx)
                for i in idx[: 10 - len(shown)]:
                    x = float(np.array(c0 + i, np.uint32).view(np.float32))
                    shown.append(f"{x!r}: device {g[i].decode()!r}, %g {w[i].decode()!r}")
            print(f"  {checked:>11} values, {bad} mismatches, {time.time() - t0:.0f} s", flush=True)
    print(f"checked {checked} float32 values in [1e-4f, 1e6f): {bad} mismatches")
    for s in shown:
        print("  " + s)
    ctx.close()
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
