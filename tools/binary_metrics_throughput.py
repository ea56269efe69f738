"""Time BinaryClassificationMetrics on the GPU (`srs_binary_metrics_create_device` / `_create_host`).

    python tools/binary_metrics_throughput.py [--repeats N] [--warmup W] [--out DIR]

Workloads (DESIGN.md section 4.22): n = 10^6, 10^7 and 10^8 seeded pairs - float32 uniform scores in [0, 1) (nearly
all distinct) with labels drawn at the score's probability - as one set and as 10^4 sets of seeded uneven sizes.
Each is timed on the device path (scores and labels already in HBM, as CTRModel leaves them); the one-set workloads
also on the host path (float64 arrays in host memory, uploaded by the call).  Times are the host clock around each
synchronous call after --warmup calls: median, min and max of --repeats.  A separate profiled call of each
device-path workload splits the kernel time into the radix sorts, the run scans (DeviceScan / DeviceSelect) and the
library's own kernels (keys, runs, points, areas).  The GPU's name, power limit and maximum SM clock are read in
the same run.  Prints one JSON document; --out also writes it to DIR/binary_metrics_throughput.json.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "unavailable (%s)" % e


def offsets(n, n_sets, seed):
    if n_sets == 1:
        return None
    w = np.random.default_rng(seed).random(n_sets) + 0.05
    cut = np.floor(np.cumsum(w) / w.sum() * n).astype(np.int64)
    cut[-1] = n
    off = np.concatenate([[0], cut])
    off[1:] = np.maximum(off[1:], np.arange(1, n_sets + 1))               # every set non-empty
    return off


def timed(fn, warmup, repeats):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return {"median_s": float(np.median(ts)), "min_s": min(ts), "max_s": max(ts)}


def kernel_split(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {"sort": 0.0, "scan_select": 0.0, "library": 0.0, "other": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        name = e.key
        if t <= 0 or "Memcpy" in name or "Memset" in name:
            continue
        if "RadixSort" in name or "Onesweep" in name or "radix" in name.lower():
            split["sort"] += t / 1e6
        elif "DeviceScan" in name or "DeviceSelect" in name or "Select" in name or "Scan" in name:
            split["scan_select"] += t / 1e6
        elif "bm_" in name:
            split["library"] += t / 1e6
        else:
            split["other"] += t / 1e6
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out")
    ap.add_argument("--sizes", default="1000000,10000000,100000000")
    a = ap.parse_args()
    import torch
    from sparrowrecsys_b200.evaluation import BinaryClassificationMetrics
    res = {"gpu": gpu_info(), "workloads": []}
    for n in [int(x) for x in a.sizes.split(",")]:
        g = torch.Generator(device="cuda").manual_seed(n)
        s = torch.rand(n, device="cuda", generator=g)
        y = (torch.rand(n, device="cuda", generator=g) < s).to(torch.int32)
        for n_sets in (1, 10_000):
            off = offsets(n, n_sets, n)

            def dev():
                with BinaryClassificationMetrics(s, y, 0, off) as m:
                    return m.summary(0).thresholds
            row = {"n": n, "sets": n_sets, "path": "device", **timed(dev, a.warmup, a.repeats)}
            row["pairs_per_s"] = n / row["median_s"]
            row["kernel_s"] = kernel_split(dev)
            res["workloads"].append(row)
            print(json.dumps(row), file=sys.stderr)
        hs, hy = s.double().cpu().numpy(), y.double().cpu().numpy()

        def host():
            with BinaryClassificationMetrics(hs, hy) as m:
                return m.summary(0).thresholds
        row = {"n": n, "sets": 1, "path": "host", **timed(host, a.warmup, a.repeats)}
        row["pairs_per_s"] = n / row["median_s"]
        res["workloads"].append(row)
        print(json.dumps(row), file=sys.stderr)
        del s, y, hs, hy
        torch.cuda.empty_cache()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "binary_metrics_throughput.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
