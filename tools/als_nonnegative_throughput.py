"""Time nonnegative ALS (`collab.als(..., nonnegative=True)`) on the GPU next to the Cholesky fit, and count the NNLS
iterations per entity, against the C oracle's single-threaded run.

    python tools/als_nonnegative_throughput.py [--skip-fixture] [--skip-synthetic] [--out DIR]

Two workloads at the script's settings (rank 10, regParam 0.01, explicit feedback): the fixture
(tests/golden/featureeng_ratings.npz, 203 150 ratings) and the seeded synthetic ML-20M-sized set of
tools/featureeng_throughput.py (20 000 263 ratings, 138 494 users, 27 278 movies).  For each, in the same call:
- the fit per iteration, nonnegative and Cholesky: the wall time of a whole synchronous call at 1 and 3 iterations,
  their difference over 2 (the upload, the layout sorts and the copies cancel);
- the NNLS iterations per entity of the first iteration's two half-steps (mean, max and how many ran to iterMax =
  max(400, 20 rank)), counted by the C oracle, whose factors are checked bit-equal to the device's;
- the C oracle's time for that iteration.
The GPU's name, power limit and maximum SM clock are read in the same call.  Prints one JSON document; --out also
writes it to DIR/als_nonnegative_throughput.json.
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

from als_throughput import gpu_info, timed  # noqa: E402


def _dist(it, k):
    from oracle import als_nnls as N
    return {"entities": int(len(it)), "mean": round(float(it.mean()), 3), "max": int(it.max()),
            "at_iter_max": int(np.sum(it == N.iter_max(k)))}


def workload(name, r, repeats, rank=10):
    from oracle import als as A
    from oracle import als_cext as X
    from oracle import als_nnls_cext as XN
    from sparrowrecsys_b200 import collab
    r = {"userId": np.asarray(r["userId"], np.int32), "movieId": np.asarray(r["movieId"], np.int32),
         "rating": np.asarray(r["rating"], np.float32)}
    n1, _ = timed(lambda: collab.als(r, rank=rank, max_iter=1, nonnegative=True), repeats)
    n3, _ = timed(lambda: collab.als(r, rank=rank, max_iter=3, nonnegative=True), repeats)
    c1, _ = timed(lambda: collab.als(r, rank=rank, max_iter=1), repeats)
    c3, _ = timed(lambda: collab.als(r, rank=rank, max_iter=3), repeats)
    per_nn, per_ch = (n3 - n1) / 2, (c3 - c1) / 2
    res = {"workload": name, "ratings": int(len(r["userId"])), "rank": rank,
           "nonnegative_call_seconds_1_iteration": round(n1, 4), "nonnegative_call_seconds_3_iterations": round(n3, 4),
           "nonnegative_seconds_per_iteration": round(per_nn, 5), "cholesky_seconds_per_iteration": round(per_ch, 5),
           "nonnegative_over_cholesky": round(per_nn / per_ch, 2) if per_ch > 0 else None}
    print(json.dumps(res), flush=True)

    uids, mids, by_movie, by_user = A.layouts(r["userId"], r["movieId"], r["rating"])
    U = X.init_user_factors(uids, rank, 0)
    it_m, it_u = np.zeros(len(mids), np.int32), np.zeros(len(uids), np.int32)
    t0 = time.perf_counter()
    M, _ = XN.solve_half(by_movie, U, uids, rank, 0.01, None, it_m)
    U1, _ = XN.solve_half(by_user, M, mids, rank, 0.01, None, it_u)
    res["c_oracle_nonnegative_seconds_per_iteration"] = round(time.perf_counter() - t0, 4)
    res["nnls_iterations_movies"] = _dist(it_m, rank)
    res["nnls_iterations_users"] = _dist(it_u, rank)
    dev = collab.als(r, rank=rank, max_iter=1, nonnegative=True)
    res["one_iteration_equals_c_oracle"] = bool(np.array_equal(dev.user_factors.view(np.int32), U1.view(np.int32))
                                                and np.array_equal(dev.item_factors.view(np.int32),
                                                                   M.view(np.int32)))
    res["fit_speedup_vs_c_oracle"] = round(res["c_oracle_nonnegative_seconds_per_iteration"] / per_nn, 1) \
        if per_nn > 0 else None
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--skip-synthetic", action="store_true")
    ap.add_argument("--skip-fixture", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool measures the GPU and has no CPU fallback")
    from sparrowrecsys_b200 import collab
    from test_als_oracle import fixture_ratings
    doc = {"gpu": gpu_info(), "workloads": []}
    print(json.dumps({"gpu": doc["gpu"]}), flush=True)
    warm = {k: v[:5000] for k, v in fixture_ratings().items()}
    collab.als(warm, max_iter=1, nonnegative=True)                     # warm-up: module load, context
    collab.als(warm, max_iter=1)
    if not a.skip_fixture:
        doc["workloads"].append(workload("fixture", fixture_ratings(), a.repeats))
    if not a.skip_synthetic:
        from featureeng_throughput import synthetic_ml20m
        doc["workloads"].append(workload("synthetic ML-20M", synthetic_ml20m()[0], 1))
    doc["gpu_after"] = gpu_info()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "als_nonnegative_throughput.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
