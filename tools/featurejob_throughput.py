"""Time the FeatureEngineering job (`featureeng.feature_engineering`) and the sample split (`split_samples`) on
the GPU against the numpy oracle on the host.

    python tools/featurejob_throughput.py [--repeats 5] [--out DIR]

Workloads: the fixture (tests/golden/featureeng_ratings.npz, 203 150 ratings; the split runs on its build_samples
rows) and the synthetic ML-20M-sized set of tools/featureeng_throughput.py (20 000 263 ratings, 27 278 movies; the
split runs on its rating rows, as many rows as ML-20M's samples).  The device time is the wall clock of the whole
synchronous call: host checks, tokenising, uploads, every kernel, copies back and the row gathers.  Every device
run is checked bit for bit against the first and the first against the oracle.  Prints one JSON line per
measurement, with the GPU's name and power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _bits(x):
    x = np.asarray(x)
    return x.view(np.int64) if x.dtype == np.float64 else x


def _equal(a, b):
    if isinstance(a, dict):
        return all(_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    if isinstance(a, (int, float, str)):
        return a == b
    return np.array_equal(_bits(a), _bits(b))


def timed(fn, repeats):
    fn()                                                            # warm-up: module load, allocator
    times, first = [], None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t0)
        if first is None:
            first = out
        assert _equal(out, first), "device runs differ"
    return first, times


def oracle_job(ratings, movies):
    from oracle import feature_job as J
    ids, n, avg, var, bucket, scaled, splits = J.feature_engineering(
        ratings["movieId"], (np.asarray(ratings["rating"]) * 2).astype(np.int64))
    labels, counts, mids, off, ind = J.multi_hot(movies["movieId"], movies["genres"])
    return {"movieId": ids, "ratingCount": n, "avgRating": avg, "ratingVar": var, "ratingCountBucket": bucket,
            "scaleAvgRating": scaled, "splits": splits}, (labels, mids, off.astype(np.int32), ind)


def run_job(name, ratings, movies, repeats):
    from sparrowrecsys_b200 import featureeng as FE
    first, times = timed(lambda: FE.feature_engineering(ratings, movies), repeats)
    t0 = time.perf_counter()
    mf, (labels, mids, off, ind) = oracle_job(ratings, movies)
    oracle_s = time.perf_counter() - t0
    mh = first["multi_hot"]
    ok = _equal({k: first["movie_features"][k] for k in mf}, mf) and mh["labels"] == labels and \
        _equal([mh["movieId"], mh["offsets"], mh["indices"]], [mids, off, ind])
    return {"workload": name, "call": "feature_engineering", "ratings": int(len(ratings["movieId"])),
            "movies": int(len(movies["movieId"])), "gpu_s_median": float(np.median(times)),
            "gpu_s_min": float(np.min(times)), "gpu_s_max": float(np.max(times)), "repeats": repeats,
            "oracle_s": oracle_s, "bit_equal_to_oracle": bool(ok), "speedup": oracle_s / float(np.median(times))}


def run_split(name, samples, repeats):
    from oracle import feature_job as J
    from sparrowrecsys_b200 import featureeng as FE
    n = len(samples["movieId"])
    first, times = timed(lambda: FE.split_samples(samples, seed=1), repeats)
    t0 = time.perf_counter()
    parts = [{k: np.asarray(v)[r] for k, v in samples.items()} for r in J.split_samples(n, 1)]
    oracle_s = time.perf_counter() - t0
    return {"workload": name, "call": "split_samples", "rows": n, "sampled": int(sum(len(p["movieId"]) for p in first)),
            "gpu_s_median": float(np.median(times)), "gpu_s_min": float(np.min(times)),
            "gpu_s_max": float(np.max(times)), "repeats": repeats, "oracle_s": oracle_s,
            "bit_equal_to_oracle": bool(_equal(first, parts)), "speedup": oracle_s / float(np.median(times))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from featureeng_throughput import gpu_info, synthetic_ml20m
    from sparrowrecsys_b200 import featureeng as FE
    from test_featureeng_oracle import fixture_inputs
    info = gpu_info()
    results = []
    r, m = fixture_inputs()
    results.append(run_job("ratings.csv, users 1..5000", r, m, a.repeats))
    results.append(run_split("ratings.csv, users 1..5000", FE.build_samples(r, m), a.repeats))
    r, m = synthetic_ml20m()
    results.append(run_job("synthetic ML-20M", r, m, a.repeats))
    results.append(run_split("synthetic ML-20M", r, a.repeats))
    for res in results:
        res["gpu"] = info
        print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "featurejob_throughput.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
