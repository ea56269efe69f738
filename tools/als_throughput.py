"""Time ALS on the GPU (`collab.als`, `AlsModel.recommend_for_all_users`) against the C oracle's single-threaded run.

    python tools/als_throughput.py [--skip-fixture] [--skip-synthetic] [--oracle-sources 2000] [--out DIR]

Two workloads at the script's settings (rank 10, regParam 0.01): the fixture (tests/golden/featureeng_ratings.npz,
203 150 ratings, all of them trained on) and the seeded synthetic ML-20M-sized set of
tools/featureeng_throughput.py (20 000 263 ratings, 138 494 users, 27 278 movies).  For each: the wall time of a
whole `als` call at 1 and 3 iterations (host clock around a synchronous call) and the time per iteration as their
difference over 2, so the upload, the layout sorts and the copies cancel; the wall time of
`recommend_for_all_users(10)`; and the C oracle's time for one iteration (its two half-steps on layouts built
beforehand) and for recommend_for_all_users(10).  On the synthetic set the oracle's recommend time is taken on the
first --oracle-sources users and scaled to all of them (reported as such).  The GPU's name and power limit are read
in the same call.  Prints one JSON document; --out also writes it to DIR/als_throughput.json.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "unavailable (%s)" % e
    return out


def timed(f, repeats):
    ts = []
    out = None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = f()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def workload(name, r, repeats, oracle_sources):
    from oracle import als as A
    from oracle import als_cext as X
    from sparrowrecsys_b200 import collab
    r = {"userId": np.asarray(r["userId"], np.int32), "movieId": np.asarray(r["movieId"], np.int32),
         "rating": np.asarray(r["rating"], np.float32)}
    t1, _ = timed(lambda: collab.als(r, max_iter=1), repeats)
    t3, model = timed(lambda: collab.als(r, max_iter=3), repeats)
    per_iter = (t3 - t1) / 2
    t_rec, (uids, ids, sc) = timed(lambda: model.recommend_for_all_users(10), repeats)
    res = {"workload": name, "ratings": int(len(r["userId"])), "users": int(len(model.user_ids)),
           "movies": int(len(model.item_ids)), "call_seconds_1_iteration": round(t1, 4),
           "call_seconds_3_iterations": round(t3, 4), "seconds_per_iteration": round(per_iter, 5),
           "recommend_all_users_10_seconds": round(t_rec, 5),
           "recommend_pairs_per_second": round(len(model.user_ids) * len(model.item_ids) / t_rec)}
    print(json.dumps(res), flush=True)
    uids_o, mids_o, by_movie, by_user = A.layouts(r["userId"], r["movieId"], r["rating"])
    U = X.init_user_factors(uids_o, 10, 0)
    t0 = time.perf_counter()
    M, _ = X.solve_half(by_movie, U, 10, 0.01)
    X.solve_half(by_user, M, 10, 0.01)
    res["c_oracle_seconds_per_iteration"] = round(time.perf_counter() - t0, 4)
    ns = min(oracle_sources, len(model.user_ids))
    t0 = time.perf_counter()
    oi, os_ = X.recommend(model.user_factors[:ns], model.item_ids, model.item_factors, 10)
    t_o = (time.perf_counter() - t0) * len(model.user_ids) / ns
    res["c_oracle_recommend_all_users_10_seconds"] = round(t_o, 3)
    res["c_oracle_recommend_sources_timed"] = ns
    res["recommend_head_equals_c_oracle"] = bool(np.array_equal(oi, ids[:ns]) and
                                                 np.array_equal(os_.view(np.int32), sc[:ns].view(np.int32)))
    res["fit_speedup_vs_c_oracle"] = round(res["c_oracle_seconds_per_iteration"] / per_iter, 1) if per_iter > 0 \
        else None
    res["recommend_speedup_vs_c_oracle"] = round(t_o / t_rec, 1)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--oracle-sources", type=int, default=2000)
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
    collab.als({k: v[:5000] for k, v in fixture_ratings().items()}, max_iter=1)   # warm-up: module load, context
    if not a.skip_fixture:
        fx = fixture_ratings()
        doc["workloads"].append(workload("fixture", fx, a.repeats, len(np.unique(fx["userId"]))))
    if not a.skip_synthetic:
        from featureeng_throughput import synthetic_ml20m
        doc["workloads"].append(workload("synthetic ML-20M", synthetic_ml20m()[0], 1, a.oracle_sources))
    doc["gpu_after"] = gpu_info()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "als_throughput.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
