"""Time implicit-feedback ALS (`collab.als(..., implicit_prefs=True)`) and `collab.ranking_metrics` on the GPU against
the C oracles' single-threaded runs.

    python tools/als_implicit_throughput.py [--skip-fixture] [--skip-synthetic] [--out DIR]

Two workloads at the script's settings (rank 10, regParam 0.01, alpha 1.0): the fixture
(tests/golden/featureeng_ratings.npz, 203 150 ratings) and the seeded synthetic ML-20M-sized set of
tools/featureeng_throughput.py (20 000 263 ratings, 138 494 users, 27 278 movies).  For each:
- the fit per iteration: the wall time of a whole synchronous call at 1 and 3 iterations, their difference over 2
  (the upload, the layout sorts and the copies cancel), next to the explicit fit's measured the same way;
- YtY's share: a separate one-iteration call under torch.profiler, the device time of als_yty_kernel and
  als_yty_merge_kernel over that of every als_* kernel of the iteration loop;
- the ranking metrics at k = 10 of the 0.8 / 0.2 split's model (the call's wall time, predictions given);
- the C oracles: one implicit iteration on layouts built beforehand, and the ranking metrics, with their outputs
  checked equal to the device's.
The GPU's name, power limit and maximum SM clock are read in the same call.  Prints one JSON document; --out also
writes it to DIR/als_implicit_throughput.json.
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


def yty_share(r):
    """(YtY kernels' device seconds, all ALS kernels' device seconds) of a one-iteration implicit fit."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from sparrowrecsys_b200 import collab
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        collab.als(r, max_iter=1, implicit_prefs=True)
        torch.cuda.synchronize()
    yty = total = 0.0
    for ev in prof.key_averages():
        name = ev.key
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if "als_yty" in name:
            yty += t
        if "als_yty" in name or "als_solve_kernel" in name:
            total += t
    return yty * 1e-6, total * 1e-6


def workload(name, r, repeats):
    from oracle import als as A
    from oracle import als_cext as X
    from oracle import als_implicit_cext as XI
    from sparrowrecsys_b200 import collab
    r = {"userId": np.asarray(r["userId"], np.int32), "movieId": np.asarray(r["movieId"], np.int32),
         "rating": np.asarray(r["rating"], np.float32)}
    t1, _ = timed(lambda: collab.als(r, max_iter=1, implicit_prefs=True), repeats)
    t3, _ = timed(lambda: collab.als(r, max_iter=3, implicit_prefs=True), repeats)
    e1, _ = timed(lambda: collab.als(r, max_iter=1), repeats)
    e3, _ = timed(lambda: collab.als(r, max_iter=3), repeats)
    per_iter, per_iter_e = (t3 - t1) / 2, (e3 - e1) / 2
    yty_s, kern_s = yty_share(r)
    res = {"workload": name, "ratings": int(len(r["userId"])), "implicit_call_seconds_1_iteration": round(t1, 4),
           "implicit_call_seconds_3_iterations": round(t3, 4), "implicit_seconds_per_iteration": round(per_iter, 5),
           "explicit_seconds_per_iteration": round(per_iter_e, 5),
           "yty_device_seconds_per_iteration": round(yty_s, 6), "als_kernels_device_seconds_per_iteration":
           round(kern_s, 6), "yty_share_of_kernel_time": round(yty_s / kern_s, 4) if kern_s else None}
    print(json.dumps(res), flush=True)

    tr, te = collab.random_split(len(r["userId"]), (0.8, 0.2), 0)
    model = collab.als({k: v[tr] for k, v in r.items()}, implicit_prefs=True)
    users, rows, labels = model.ranking_queries({k: v[te] for k, v in r.items()})
    _, pred, _ = model.recommend_for_user_subset(users, 10)
    t_rm, got = timed(lambda: collab.ranking_metrics(pred, labels, 10), repeats)
    t0 = time.perf_counter()
    means, _ = XI.ranking_metrics(pred, labels[0], labels[1], 10)
    t_rm_o = time.perf_counter() - t0
    res.update({"ranking_queries": int(len(users)), "ranking_labels": int(labels[0][-1]),
                "ranking_metrics_seconds": round(t_rm, 5), "c_oracle_ranking_metrics_seconds": round(t_rm_o, 4),
                "ranking_metrics_equal_c_oracle": [got["precision_at_k"], got["ndcg_at_k"],
                                                   got["mean_average_precision"]] == means.tolist(),
                "precision_at_10": got["precision_at_k"], "ndcg_at_10": got["ndcg_at_k"],
                "map": got["mean_average_precision"]})
    print(json.dumps(res), flush=True)

    uids, mids, by_movie, by_user = A.layouts(r["userId"], r["movieId"], r["rating"])
    U = X.init_user_factors(uids, 10, 0)
    t0 = time.perf_counter()
    M, _ = XI.solve_half(by_movie, U, uids, 10, 0.01, 1.0)
    U1, _ = XI.solve_half(by_user, M, mids, 10, 0.01, 1.0)
    res["c_oracle_implicit_seconds_per_iteration"] = round(time.perf_counter() - t0, 4)
    dev = collab.als(r, max_iter=1, implicit_prefs=True)
    res["one_iteration_equals_c_oracle"] = bool(np.array_equal(dev.user_factors.view(np.int32), U1.view(np.int32)))
    res["fit_speedup_vs_c_oracle"] = round(res["c_oracle_implicit_seconds_per_iteration"] / per_iter, 1) \
        if per_iter > 0 else None
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
    collab.als(warm, max_iter=1, implicit_prefs=True)                  # warm-up: module load, context
    collab.ranking_metrics([[1, 2]], [[1]], 10)
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
        with open(os.path.join(a.out, "als_implicit_throughput.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
