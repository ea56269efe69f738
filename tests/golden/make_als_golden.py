"""Regenerate tests/golden/als_fit.json: the reference's CollaborativeFiltering sequence run by the C oracle on the
fixture ratings (featureeng_ratings.npz), at the script's settings (split 0.8 / 0.2, rank 10, maxIter 5, regParam
0.01), for seeds 0 and 1 (the split and the factors use the same seed).

    python tests/golden/make_als_golden.py [REFERENCE_ROOT]

With the root of a SparrowRecSys checkout it also runs the whole of its ratings.csv and prints the RMSE that
DESIGN.md section 4.13 quotes.  Records, per seed: the RMSE (a double, written with repr so it reads back exactly),
the split's sizes, the kept test rows, and the head of recommendForAllUsers(10) / recommendForAllItems(10).
"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import als_cext as X  # noqa: E402
from sparrowrecsys_b200 import collab  # noqa: E402

SEEDS = (0, 1)


def script(r, seed):
    """The job's sequence with the C oracle: (model, rmse, n_train, kept test rows)."""
    tr, te = collab.random_split(len(r["userId"]), (0.8, 0.2), seed)
    uids, uf, mids, mf = X.fit(r["userId"][tr], r["movieId"][tr], r["rating"][tr], rank=10, max_iter=5,
                               reg_param=0.01, seed=seed)
    model = collab.AlsModel(uids, uf, mids, mf)
    test = {k: v[te] for k, v in r.items()}
    kept, pred = model.transform(test)
    return model, collab.rmse(test["rating"][kept], pred), len(tr), len(te), kept


def main():
    z = np.load(os.path.join(HERE, "featureeng_ratings.npz"))
    r = {"userId": z["userId"].astype(np.int32), "movieId": z["movieId"].astype(np.int32),
         "rating": (z["half"] / 2.0).astype(np.float32)}
    doc = {"settings": {"split": [0.8, 0.2], "rank": 10, "max_iter": 5, "reg_param": 0.01}, "seeds": {}}
    for seed in SEEDS:
        model, rmse, n_train, n_test, kept = script(r, seed)
        ui, us = X.recommend(model.user_factors[:3], model.item_ids, model.item_factors, 10)
        mi, ms = X.recommend(model.item_factors[:3], model.user_ids, model.user_factors, 10)
        doc["seeds"][str(seed)] = {
            "rmse": rmse, "n_train": n_train, "n_test": n_test, "n_kept": int(len(kept)),
            "kept_checksum": int(np.sum(kept.astype(np.int64) * (np.arange(len(kept)) % 7 + 1))),
            "n_users": int(len(model.user_ids)), "n_movies": int(len(model.item_ids)),
            "user_recs_head": {"users": model.user_ids[:3].tolist(), "ids": ui.tolist(),
                               "scores": [[float(v) for v in row] for row in us]},
            "movie_recs_head": {"movies": model.item_ids[:3].tolist(), "ids": mi.tolist(),
                                "scores": [[float(v) for v in row] for row in ms]}}
        print("seed %d: rmse %r, %d kept of %d" % (seed, rmse, len(kept), n_test))
    with open(os.path.join(HERE, "als_fit.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    if len(sys.argv) > 1:
        from sparrowrecsys_b200.featureeng import load_ratings_csv
        path = os.path.join(sys.argv[1], "src", "main", "resources", "webroot", "sampledata", "ratings.csv")
        full = load_ratings_csv(path)
        full["rating"] = full["rating"].astype(np.float32)
        t0 = time.perf_counter()
        _, rmse, n_train, n_test, kept = script(full, 0)
        print("whole ratings.csv, seed 0: %d ratings, rmse %r over %d of %d test rows (%.1f s)"
              % (len(full["userId"]), rmse, len(kept), n_test, time.perf_counter() - t0))


if __name__ == "__main__":
    main()
