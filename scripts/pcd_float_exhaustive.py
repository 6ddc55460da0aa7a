#!/usr/bin/env python3
"""Every one of the 2^32 float bit patterns through the host build of the PCD float formatter
(gem_b200/csrc/gem_pcdfmt.h, the code gem_pcd_format runs on the device) against glibc's snprintf("%.8g") -- "nan" for
every NaN, as PCL's ASCII writer prints it.  Also checks that no value is longer than GEM_PCD_VALUE_MAX (14) characters
and that the formatter's length function agrees with what it prints.

    python scripts/pcd_float_exhaustive.py [--jobs N] [--chunks 4096]

Spreads the range over N processes (default: every core) and prints one JSON line {patterns, mismatches, first, seconds,
jobs}; exits non-zero on a mismatch."""
from __future__ import annotations

import argparse
import json
import multiprocessing as mp
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pcd_oracle  # noqa: E402


def _run(span):
    lo, hi = span
    return pcd_oracle.fmt_compare_range(lo, hi)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--jobs", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--chunks", type=int, default=4096)
    a = ap.parse_args()
    pcd_oracle.load_fmt()   # build once before the workers fork
    total = 1 << 32
    step = total // a.chunks
    spans = [(i * step, total if i == a.chunks - 1 else (i + 1) * step) for i in range(a.chunks)]
    t0 = time.time()
    bad, first = 0, None
    with mp.get_context("fork").Pool(a.jobs) as pool:
        for k, f in pool.imap(_run, spans):
            if k and first is None:
                first = f
            bad += k
    res = {"patterns": total, "mismatches": bad, "first": None if first is None else f"0x{first:08x}",
           "seconds": round(time.time() - t0, 1), "jobs": a.jobs}
    print(json.dumps(res))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
