"""Time the batched ALS fit of a cross-validation (`collab.als_folds`, one `srs_als_fit_folds_host` call for every
fold x grid model) against a loop of single fits (`collab.als`, one `srs_als_fit_host` per model) over the same
models, and check that both give the same bits.

    python tools/als_cv_throughput.py [--skip-fixture] [--skip-synthetic] [--repeats 3] [--out DIR]

Two workloads at rank 10, maxIter 5: the reference script's CV step on the fixture (the 0.2 test part of
tests/golden/featureeng_ratings.npz, 40 601 ratings, 10 folds x regParam [0.01]: 10 models) and the seeded synthetic
ML-20M-sized set of tools/featureeng_throughput.py (20 000 263 ratings, 5 folds x regParam [0.01, 0.1]: 10 models).
Times are host wall clock around synchronous calls, the median of --repeats (1 on the synthetic set), after a
warm-up call.  The loop's training subsets are cut beforehand and not timed.  The GPU's name and power limit are
read in the same run.  Prints one JSON document; --out also writes it to DIR/als_cv_throughput.json.
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


def workload(name, r, num_folds, regs, repeats):
    from sparrowrecsys_b200 import collab
    r = {"userId": np.asarray(r["userId"], np.int32), "movieId": np.asarray(r["movieId"], np.int32),
         "rating": np.asarray(r["rating"], np.float32)}
    fold = collab.fold_ids(len(r["userId"]), num_folds, seed=0)
    models = [dict(rank=10, max_iter=5, reg_param=reg, exclude_fold=f) for f in range(num_folds) for reg in regs]
    subsets = [{c: v[fold != f] for c, v in r.items()} for f in range(num_folds)]

    def loop():
        return [collab.als(subsets[m["exclude_fold"]], rank=10, max_iter=5, reg_param=m["reg_param"])
                for m in models]

    t_batch, batched = timed(lambda: collab.als_folds(r, fold, num_folds, models), repeats)
    t_loop, single = timed(loop, repeats)
    same = all(np.array_equal(a.user_ids, b.user_ids) and np.array_equal(a.item_ids, b.item_ids) and
               np.array_equal(a.user_factors.view(np.int32), b.user_factors.view(np.int32)) and
               np.array_equal(a.item_factors.view(np.int32), b.item_factors.view(np.int32))
               for a, b in zip(batched, single))
    res = {"workload": name, "ratings": int(len(r["userId"])), "folds": num_folds, "reg_params": list(regs),
           "models": len(models), "batched_seconds": round(t_batch, 4), "loop_seconds": round(t_loop, 4),
           "batched_speedup": round(t_loop / t_batch, 2), "batched_equals_loop": bool(same)}
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
    fx = fixture_ratings()
    warm = {k: v[:5000] for k, v in fx.items()}             # module load, context
    collab.als_folds(warm, collab.fold_ids(5000, 2), 2, [dict(rank=10, max_iter=1, reg_param=0.01, exclude_fold=0)])
    collab.als(warm, max_iter=1)
    if not a.skip_fixture:
        _, te = collab.random_split(len(fx["userId"]), (0.8, 0.2), 0)
        test = {k: v[te] for k, v in fx.items()}
        doc["workloads"].append(workload("fixture CV step (10 folds x [0.01])", test, 10, [0.01], a.repeats))
    if not a.skip_synthetic:
        from featureeng_throughput import synthetic_ml20m
        doc["workloads"].append(workload("synthetic ML-20M (5 folds x [0.01, 0.1])", synthetic_ml20m()[0], 5,
                                         [0.01, 0.1], 1))
    doc["gpu_after"] = gpu_info()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "als_cv_throughput.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
