"""Time of the PCD writer (DESIGN.md f13) on clouds of 1 M and 10 M harvest-like PointXYZRGBICT records, beside the C
oracle (a restatement of PCL's writeASCII, one snprintf per value) on one host thread.

- device format: CUDA events on the library's stream around one gem_pcd_format call into a device buffer that holds the
  result (the call is host-synchronous: the interval holds its synchronisations), median of CALLS after WARM, for ASCII
  and binary; output bytes and output GB/s;
- end to end: ElevationMap.save_pcd from device records and from host records into a file under the output directory
  ($GEM_BENCH_OUT, else a temporary directory; never the tree itself), host wall clock, one run each;
- the oracle's ASCII data section for the 1 M cloud on one host thread, one run; every device output of the 1 M cloud is
  checked equal to the oracle's, and the 10 M cloud's against the formatter's host build.

Prints one JSON line with the GPU name, SM clock and power limit read by nvidia-smi in the same run (also written to
$GEM_BENCH_OUT/pcd_bench.json when that is set)."""
import json
import os
import subprocess
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import gem_b200  # noqa: E402
import pcd_cases  # noqa: E402
import pcd_oracle  # noqa: E402

WARM, CALLS = 3, 20


def gpu_info():
    q = "name,clocks.sm,clocks.max.sm,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:   # the numbers are then reported without the card's state
        return {"error": str(e)}


def device_ms(g, d, binary, out):
    st = g.torch_stream()
    times = []
    for i in range(WARM + CALLS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        res = g.format_pcd(d, binary=binary, out=out)
        e1.record(st)
        e1.synchronize()
        if i >= WARM:
            times.append(e0.elapsed_time(e1))
    return float(np.median(times)), min(times), max(times), res


def main():
    if not torch.cuda.is_available():
        raise SystemExit("pcd_bench: no GPU")
    keep = os.environ.get("GEM_BENCH_OUT")
    outdir = keep or tempfile.mkdtemp(prefix="gem_pcd_bench_")
    os.makedirs(outdir, exist_ok=True)
    g = gem_b200.ElevationMap(64, 0.1, compat_box_filter=False, device=0)
    res = {"gpu": gpu_info(), "warm": WARM, "calls": CALLS, "clouds": {}}
    for n in (1_000_000, 10_000_000):
        rec = pcd_cases.harvest_like(n, 1)
        host = rec.view(np.float32)
        d = torch.from_numpy(host).to("cuda:0")
        out = torch.empty(n * gem_b200._lib.PCD_LINE_MAX, dtype=torch.uint8, device="cuda:0")
        row = {}
        for binary in (False, True):
            med, lo, hi, data = device_ms(g, d, binary, out)
            got = data.cpu().numpy().tobytes()
            if n == 1_000_000:
                ok = got == pcd_oracle.data(rec, 1 if binary else 0)
            else:
                ok = got == (pcd_oracle.fmt_ascii(rec) if not binary else pcd_oracle.py_data(rec, 1))
            key = "binary" if binary else "ascii"
            row[key] = {"device_ms": round(med, 3), "device_ms_min": round(lo, 3), "device_ms_max": round(hi, 3),
                        "bytes": len(got), "GB_per_s": round(len(got) / med / 1e6, 2), "equal": bool(ok)}
            for src_name, src in (("device", d), ("host", host)):
                path = os.path.join(outdir, f"pcd_bench_{n}_{key}_{src_name}.pcd")
                t0 = time.perf_counter()
                size = g.save_pcd(path, src, binary=binary)
                row[key][f"save_{src_name}_s"] = round(time.perf_counter() - t0, 3)
                row[key]["file_bytes"] = size
                os.remove(path)
        if n == 1_000_000:
            t0 = time.perf_counter()
            pcd_oracle.data(rec, 0)
            row["ascii"]["oracle_1thread_s"] = round(time.perf_counter() - t0, 3)
        res["clouds"][str(n)] = row
        del d, out
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if keep:
        with open(os.path.join(outdir, "pcd_bench.json"), "w") as f:
            f.write(line + "\n")
    else:
        shutil.rmtree(outdir, True)


if __name__ == "__main__":
    main()
