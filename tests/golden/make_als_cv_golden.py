"""Regenerate tests/golden/als_cv.json: the last step of the reference's CollaborativeFiltering job,
`CrossValidator(ALS, RegressionEvaluator("rmse"), regParam grid [0.01], numFolds 10).fit(test)`, run by the C
oracle (oracle/als_cv.py over oracle/als_c.c) on the fixture ratings (featureeng_ratings.npz): `test` is the 0.2 part
of the seed-0 split, the folds use seed 0 and every fit rank 10, maxIter 5 and ALS seed 0.

    python tests/golden/make_als_cv_golden.py

Records, per fold, the validation rows and how many of them are cold (their user or movie has no factor in that
fold's model), and the fold and average metrics with the CV's models' default cold-start strategy "nan" (the
script's run) and with "drop".  Metrics are doubles written with repr, NaN as JSON's NaN.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import als_cv as O  # noqa: E402
from sparrowrecsys_b200 import collab  # noqa: E402

GRID = [("reg_param", [0.01])]
FOLDS = 10


def script_test_split():
    z = np.load(os.path.join(HERE, "featureeng_ratings.npz"))
    r = {"userId": z["userId"].astype(np.int32), "movieId": z["movieId"].astype(np.int32),
         "rating": (z["half"] / 2.0).astype(np.float32)}
    _, te = collab.random_split(len(r["userId"]), (0.8, 0.2), 0)
    return {k: v[te] for k, v in r.items()}


def main():
    test = script_test_split()
    doc = {"settings": {"split_seed": 0, "fold_seed": 0, "num_folds": FOLDS, "grid": GRID, "rank": 10,
                        "max_iter": 5, "als_seed": 0, "metric": "rmse"}, "n_rows": int(len(test["userId"]))}
    fold = O.fold_of(len(test["userId"]), FOLDS, 0)
    doc["validation_rows"] = np.bincount(fold, minlength=FOLDS).tolist()
    for strategy in ("nan", "drop"):
        res = O.cross_validate(test, GRID, FOLDS, "rmse", strategy)
        doc["cold_rows"] = res["cold_rows"]
        doc[strategy] = {"fold_metrics": res["fold_metrics"], "avg_metrics": res["avg_metrics"],
                         "best_index": res["best_index"]}
        print("%s: avgMetrics %r, cold rows per fold %r" % (strategy, res["avg_metrics"], res["cold_rows"]))
    with open(os.path.join(HERE, "als_cv.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
