"""Regenerate tests/golden/als_nonnegative.json: the CollaborativeFiltering sequence with nonnegative = true
(`python -m sparrowrecsys_b200.collab ratings.csv --nonnegative`, with `--implicit` and with `--cv`) run by the C
oracles on the fixture ratings (featureeng_ratings.npz): split 0.8 / 0.2 at seed 0, ALS rank 10, maxIter 5,
regParam 0.01, seed 0 (alpha 1.0 when implicit); the explicit run's test RMSE with coldStartStrategy "drop", the
implicit run's RankingMetrics at k = 10 of each test user's top 10 against its test movies rated above 0, and
CrossValidator(regParam grid [0.01], numFolds 10, fold seed 0) on the test part with every fit nonnegative.

    python tests/golden/make_als_nonnegative_golden.py

Doubles are written with repr so they read back exactly; the factor and recommendation heads are the first three
rows of each run's factors and recommendForAllUsers(10) / recommendForAllItems(10).
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import als_cext as X  # noqa: E402
from oracle import als_cv as O  # noqa: E402
from oracle import als_implicit_cext as XI  # noqa: E402
from oracle import als_nnls_cext as XN  # noqa: E402
from sparrowrecsys_b200 import collab  # noqa: E402

SETTINGS = {"split": [0.8, 0.2], "seed": 0, "rank": 10, "max_iter": 5, "reg_param": 0.01, "alpha": 1.0, "k": 10,
            "cv_grid": [["reg_param", [0.01]]], "cv_folds": 10, "cv_fold_seed": 0}


def fixture():
    z = np.load(os.path.join(HERE, "featureeng_ratings.npz"))
    return {"userId": z["userId"].astype(np.int32), "movieId": z["movieId"].astype(np.int32),
            "rating": (z["half"] / 2.0).astype(np.float32)}


def heads(model):
    ui, us = X.recommend(model.user_factors[:3], model.item_ids, model.item_factors, 10)
    mi, ms = X.recommend(model.item_factors[:3], model.user_ids, model.user_factors, 10)
    return {"n_users": int(len(model.user_ids)), "n_movies": int(len(model.item_ids)),
            "user_factors_head": [[float(v) for v in row] for row in model.user_factors[:3]],
            "item_factors_head": [[float(v) for v in row] for row in model.item_factors[:3]],
            "user_recs_head": {"users": model.user_ids[:3].tolist(), "ids": ui.tolist(),
                               "scores": [[float(v) for v in row] for row in us]},
            "movie_recs_head": {"movies": model.item_ids[:3].tolist(), "ids": mi.tolist(),
                                "scores": [[float(v) for v in row] for row in ms]}}


def main():
    r = fixture()
    tr, te = collab.random_split(len(r["userId"]), (0.8, 0.2), 0)
    train = {k: v[tr] for k, v in r.items()}
    test = {k: v[te] for k, v in r.items()}
    doc = {"settings": SETTINGS, "n_train": int(len(tr)), "n_test": int(len(te))}

    model = collab.AlsModel(*XN.fit(train["userId"], train["movieId"], train["rating"], rank=10, max_iter=5,
                                    reg_param=0.01, seed=0))
    kept, pred = model.transform(test)
    doc["explicit"] = dict(heads(model), rmse=collab.rmse(test["rating"][kept], pred), n_kept=int(len(kept)))

    model = collab.AlsModel(*XN.fit(train["userId"], train["movieId"], train["rating"], rank=10, max_iter=5,
                                    reg_param=0.01, seed=0, implicit_prefs=True, alpha=1.0))
    users, rows, (off, ids) = model.ranking_queries(test)
    pred, _ = X.recommend(model.user_factors[rows], model.item_ids, model.item_factors, 10)
    means, _ = XI.ranking_metrics(pred, off, ids, 10)
    doc["implicit"] = dict(heads(model), precision_at_k=float(means[0]), ndcg_at_k=float(means[1]),
                           mean_average_precision=float(means[2]), n_queries=int(len(users)),
                           n_relevant=int(off[-1]))

    cv = O.cross_validate(test, [("reg_param", [0.01])], 10, "rmse", "nan", fit=XN.fit)
    doc["cv"] = {"avg_metrics": cv["avg_metrics"], "fold_metrics": cv["fold_metrics"], "cold_rows": cv["cold_rows"]}

    print("RMSE %r; precision@10 %r, ndcg@10 %r, MAP %r; CV avgMetrics %r"
          % (doc["explicit"]["rmse"], *(float(v) for v in means), cv["avg_metrics"]))
    with open(os.path.join(HERE, "als_nonnegative.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
