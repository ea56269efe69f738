"""Regenerate tests/golden/als_implicit.json: the CollaborativeFiltering sequence with implicitPrefs
(`python -m sparrowrecsys_b200.collab ratings.csv --implicit`) run by the C oracles on the fixture ratings
(featureeng_ratings.npz): split 0.8 / 0.2 at seed 0, ALS rank 10, maxIter 5, regParam 0.01, alpha 1.0, seed 0,
then RankingMetrics at k = 10 of each test user's top 10 against its test movies rated above 0.

    python tests/golden/make_als_implicit_golden.py

Records the three metrics (doubles, written with repr so they read back exactly), the split's and the queries'
sizes, and the head of the factors and of recommendForAllUsers(10) / recommendForAllItems(10).
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import als_cext as X  # noqa: E402
from oracle import als_implicit_cext as XI  # noqa: E402
from sparrowrecsys_b200 import collab  # noqa: E402

SETTINGS = {"split": [0.8, 0.2], "seed": 0, "rank": 10, "max_iter": 5, "reg_param": 0.01, "alpha": 1.0, "k": 10}


def script(r):
    """The --implicit sequence with the C oracles: (model, metrics [3], n_train, n_queries, n_relevant)."""
    tr, te = collab.random_split(len(r["userId"]), (0.8, 0.2), 0)
    uids, uf, mids, mf = XI.fit(r["userId"][tr], r["movieId"][tr], r["rating"][tr], rank=10, max_iter=5,
                                reg_param=0.01, alpha=1.0, seed=0)
    model = collab.AlsModel(uids, uf, mids, mf)
    test = {k: v[te] for k, v in r.items()}
    users, rows, (off, ids) = model.ranking_queries(test)
    pred, _ = X.recommend(model.user_factors[rows], model.item_ids, model.item_factors, 10)
    means, _ = XI.ranking_metrics(pred, off, ids, 10)
    return model, means, len(tr), len(users), int(off[-1])


def main():
    z = np.load(os.path.join(HERE, "featureeng_ratings.npz"))
    r = {"userId": z["userId"].astype(np.int32), "movieId": z["movieId"].astype(np.int32),
         "rating": (z["half"] / 2.0).astype(np.float32)}
    model, means, n_train, n_queries, n_relevant = script(r)
    ui, us = X.recommend(model.user_factors[:3], model.item_ids, model.item_factors, 10)
    mi, ms = X.recommend(model.item_factors[:3], model.user_ids, model.user_factors, 10)
    doc = {"settings": SETTINGS, "precision_at_k": float(means[0]), "ndcg_at_k": float(means[1]),
           "mean_average_precision": float(means[2]), "n_train": n_train, "n_queries": n_queries,
           "n_relevant": n_relevant, "n_users": int(len(model.user_ids)), "n_movies": int(len(model.item_ids)),
           "user_factors_head": [[float(v) for v in row] for row in model.user_factors[:3]],
           "item_factors_head": [[float(v) for v in row] for row in model.item_factors[:3]],
           "user_recs_head": {"users": model.user_ids[:3].tolist(), "ids": ui.tolist(),
                              "scores": [[float(v) for v in row] for row in us]},
           "movie_recs_head": {"movies": model.item_ids[:3].tolist(), "ids": mi.tolist(),
                               "scores": [[float(v) for v in row] for row in ms]}}
    print("precision@10 %r, ndcg@10 %r, MAP %r over %d queries" % (*(float(v) for v in means), n_queries))
    with open(os.path.join(HERE, "als_implicit.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
