"""Time BucketedRandomProjectionLSHModel.approx_similarity_join on the GPU (`srs_lsh_similarity_join_host`).

    python tools/lsh_join_throughput.py [--repeats N] [--warmup W] [--out DIR]

Workloads (DESIGN.md section 4.14):
1. the 881 shipped item2vec vectors joined with themselves at the reference's settings (bucket length 0.1, 3 tables,
   the default seed), threshold 0.3; the CPU oracle (oracle/lsh_join.py) is timed on this workload only;
2. 10^5 seeded N(0, 1) 64-dim float32 vectors joined with themselves, 3 tables, bucket length 0.1, threshold 8.5
   (about 8 * 10^8 candidates and a few 10^6 pairs);
3. one bucket of 20 000 x 20 000 seeded N(0, 1) 64-dim vectors, the first entry made >= 0, under the unit vector e_0
   at bucket length 10^30 (4 * 10^8 candidates), threshold 7, which keeps few pairs.
"candidates" is the work the device walks: the sum over tables of the (a, b) sharing that table's bucket, counted
on the host from the bucket ids.  Times are the host clock around each synchronous call, after --warmup calls:
median, min and max of --repeats.  The GPU's name and power limit are read in the same run.  Prints one JSON
document; --out also writes it to DIR/lsh_join_throughput.json.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "unavailable (%s)" % e
    return out


def candidates(model, xa, xb):
    """sum over tables of sum over buckets of count_A * count_B"""
    from oracle import lsh as H
    ha = H.transform(xa, model.rand_unit_vectors, model.bucket_length)
    hb = H.transform(xb, model.rand_unit_vectors, model.bucket_length)
    total = 0
    for j in range(ha.shape[1]):
        ua, ca = np.unique(ha[:, j] + 0.0, return_counts=True)
        ub, cb = np.unique(hb[:, j] + 0.0, return_counts=True)
        _, ia, ib = np.intersect1d(ua, ub, assume_unique=True, return_indices=True)
        total += int(np.sum(ca[ia].astype(np.int64) * cb[ib].astype(np.int64)))
    return total


def workload(name, model, ia, xa, ib, xb, threshold, warmup, repeats):
    for _ in range(warmup):
        model.approx_similarity_join(ia, xa, ib, xb, threshold)
    ts, out = [], None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = model.approx_similarity_join(ia, xa, ib, xb, threshold)
        ts.append(time.perf_counter() - t0)
    C = candidates(model, xa, xb)
    med = float(np.median(ts))
    return {"workload": name, "n_a": len(ia), "n_b": len(ib), "dim": xa.shape[1],
            "tables": model.rand_unit_vectors.shape[0], "bucket_length": model.bucket_length,
            "threshold": threshold, "candidates": C, "pairs": int(len(out[0])), "call_s_median": med,
            "call_s_min": float(min(ts)), "call_s_max": float(max(ts)), "repeats": repeats, "warmup": warmup,
            "candidates_per_s": C / med}, out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    from oracle import lsh_join as J
    from sparrowrecsys_b200 import embedding as E
    from test_item2vec_oracle import shipped_items

    res = {"gpu": gpu_info(), "workloads": []}
    sid, svec = shipped_items()
    m1 = E.BucketedRandomProjectionLSH().fit(svec)
    r1, out1 = workload("shipped 881 self-join, reference settings", m1, sid, svec, sid, svec, 0.3, a.warmup,
                        a.repeats)
    t0 = time.perf_counter()
    want = J.approx_similarity_join(sid, svec, sid, svec, m1.rand_unit_vectors, 0.1, 0.3)
    r1["cpu_oracle_s"] = time.perf_counter() - t0
    r1["equal_to_cpu_oracle"] = bool(all(np.array_equal(g, w) for g, w in zip(out1, want)))
    res["workloads"].append(r1)

    rng = np.random.default_rng(0)
    x = rng.standard_normal((100000, 64)).astype(np.float32)
    ids = np.arange(100000, dtype=np.int32)
    m2 = E.BucketedRandomProjectionLSH(bucket_length=0.1, num_hash_tables=3).fit(x)
    r2, _ = workload("10^5 N(0,1) 64-dim self-join", m2, ids, x, ids, x, 8.5, a.warmup, a.repeats)
    res["workloads"].append(r2)

    rng = np.random.default_rng(1)
    xa = rng.standard_normal((20000, 64)).astype(np.float32)
    xb = rng.standard_normal((20000, 64)).astype(np.float32)
    xa[:, 0], xb[:, 0] = np.abs(xa[:, 0]), np.abs(xb[:, 0])        # projections on e_0 >= 0: all in bucket 0
    i2 = np.arange(20000, dtype=np.int32)
    m3 = E.BucketedRandomProjectionLSHModel(np.eye(64)[:1], 1e30)
    r3, _ = workload("one bucket, 20 000 x 20 000, 64-dim", m3, i2, xa, i2, xb, 7.0, a.warmup, a.repeats)
    res["workloads"].append(r3)
    res["gpu_after"] = gpu_info()

    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lsh_join_throughput.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
