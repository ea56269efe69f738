"""Time the sample builder (`featureeng.build_samples` on the GPU) against the numpy oracle on the host.

    python tools/featureeng_throughput.py [--repeats 5] [--skip-large-oracle] [--out DIR]

Workloads: the ratings of the 5 000 smallest user ids of the reference's ratings.csv
(tests/golden/featureeng_ratings.npz, 203 150 ratings, up to 1 000 movie ids) and a synthetic ML-20M-sized set
(20 000 263 ratings, 138 494 users, 27 278 movies with ids spread over 1..131 262, 20 genre words).  The device time is the wall clock of the whole synchronous call: input
checks, uploads, every kernel and the copies back.  Each device run is checked bit for bit against the first, and
the first against the oracle.  Prints one JSON line per workload, with the GPU's name and power limit.
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

GENRES = ["Adventure", "Animation", "Children", "Comedy", "Fantasy", "Romance", "Drama", "Action", "Crime",
          "Thriller", "Horror", "Mystery", "Sci-Fi", "IMAX", "Documentary", "War", "Musical", "Western",
          "Film-Noir", "(no genres listed)"]


def synthetic_ml20m(seed=0, n=20000263, users=138494, movies=27278, max_id=131262):
    rng = np.random.default_rng(seed)
    ids = np.sort(np.r_[1, rng.choice(np.arange(2, max_id + 1), movies - 1, replace=False)])
    w = 1.0 / np.arange(1, movies + 1) ** 0.9                       # movie popularity, Zipf-like
    per_user = rng.pareto(1.2, users) + 1.0
    cnt = np.maximum(20, (per_user / per_user.sum() * n)).astype(np.int64)
    cnt[-1] += n - cnt.sum()
    cnt = np.maximum(cnt, 1)
    cnt[np.argmax(cnt)] -= cnt.sum() - n
    user = np.repeat(np.arange(1, users + 1, dtype=np.int32), cnt)
    movie = ids[rng.choice(movies, n, p=w / w.sum())].astype(np.int32)
    half = rng.choice(np.arange(1, 11), n, p=np.array([1, 3, 2, 7, 5, 20, 11, 27, 9, 15]) / 100.0)
    ts = rng.integers(789652009, 1427784002, n).astype(np.int32)    # 1995-01-09 .. 2015-03-31: 9 and 10 digits
    titles = ["Movie %d (%d)" % (i, y) for i, y in zip(ids.tolist(), rng.integers(1915, 2015, movies).tolist())]
    k = rng.integers(1, 5, movies)
    genres = ["|".join(GENRES[j] for j in rng.choice(len(GENRES), kk, replace=False)) for kk in k.tolist()]
    return ({"userId": user, "movieId": movie, "rating": half / 2.0, "timestamp": ts},
            {"movieId": ids.astype(np.int32), "title": titles, "genres": genres})


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                          # the measurement still stands without it
        return "unknown (%s)" % e


def same_bits(a, b):
    for c in a:
        x, y = np.asarray(a[c]), np.asarray(b[c])
        if x.dtype == np.float32:
            x, y = x.view(np.int32), y.view(np.int32)
        if x.shape != y.shape or not np.array_equal(x, y):
            return False
    return True


def run(name, ratings, movies, repeats, oracle):
    from oracle import feature_eng as F
    from sparrowrecsys_b200 import featureeng as FE
    FE.build_samples(ratings, movies, device=0)                     # warm-up: module load, allocator
    times, first = [], None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = FE.build_samples(ratings, movies, device=0)
        times.append(time.perf_counter() - t0)
        if first is None:
            first = out
        assert same_bits(out, first), "device runs differ"
    res = {"workload": name, "ratings": int(len(ratings["userId"])), "rows_kept": int(len(first["movieId"])),
           "gpu_s_median": float(np.median(times)), "gpu_s_min": float(np.min(times)),
           "gpu_s_max": float(np.max(times)), "repeats": repeats}
    if oracle:
        t0 = time.perf_counter()
        ref = F.build_samples(ratings, movies)
        res["oracle_s"] = time.perf_counter() - t0
        res["bit_equal_to_oracle"] = same_bits(first, ref)
        res["speedup"] = res["oracle_s"] / res["gpu_s_median"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--skip-large-oracle", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from test_featureeng_oracle import fixture_inputs
    info = gpu_info()
    results = []
    r, m = fixture_inputs()
    results.append(run("ratings.csv, users 1..5000", r, m, a.repeats, True))
    r, m = synthetic_ml20m()
    results.append(run("synthetic ML-20M", r, m, a.repeats, not a.skip_large_oracle))
    for res in results:
        res["gpu"] = info
        print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "featureeng_throughput.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
