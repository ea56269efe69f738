"""Restatement of the last step of the reference's CollaborativeFiltering job: Spark ML's `CrossValidator` over a
`ParamGridBuilder` grid with the `ALS` estimator and a `RegressionEvaluator` (DESIGN.md section 4.15).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT.  Spark 2.4's `CrossValidator.fit`, `MLUtils.kFold` and
`BernoulliCellSampler` are restated from memory, like oracle/als.py.  It loops a single-model fit (the C oracle's
by default) over each fold's training rows; nothing is batched or shared between models.
"""
from __future__ import annotations

import math

import numpy as np

from . import als as A
from . import als_cext as X
from .item2vec import splitmix


def fold_of(n, num_folds, seed):
    """Row i's fold (0-based): u_i = (splitmix(seed, i) >> 11) / 2^53, the same draw in every fold; fold f = 1..k
    holds lb <= u_i < ub with lb = float32(f - 1) / float32(k) and ub = float32(f) / float32(k) in float32."""
    k = int(num_folds)
    bounds = [float(np.float32(f) / np.float32(k)) for f in range(k + 1)]
    out = np.empty(n, np.int32)
    for i in range(n):
        u = (splitmix(seed & (2 ** 64 - 1), i) >> 11) * 2.0 ** -53
        out[i] = next(f for f in range(k) if bounds[f] <= u < bounds[f + 1])
    return out


def grid(pairs):
    """ParamGridBuilder.build: for each (param, values) in order, every value times every map so far."""
    maps = [{}]
    for name, values in pairs:
        maps = [dict(m, **{name: v}) for v in values for m in maps]
    return maps


def transform(model, ratings, strategy):
    """ALSModel.transform's float dot for rows whose user and movie have factors; "nan" keeps the rest as NaN,
    "drop" removes them.  Returns (labels, predictions, cold rows)."""
    uids, uf, mids, mf = model
    uidx = {int(u): i for i, u in enumerate(uids)}
    midx = {int(m): i for i, m in enumerate(mids)}
    labels, preds, cold = [], [], 0
    for u, m, r in zip(ratings["userId"].tolist(), ratings["movieId"].tolist(),
                       np.asarray(ratings["rating"], np.float32).tolist()):
        if u in uidx and m in midx:
            p = A.predict(uf[uidx[u]][None], mf[midx[m]][None])[0]
        else:
            cold += 1
            if strategy == "drop":
                continue
            p = np.float32("nan")
        labels.append(r)
        preds.append(p)
    return np.array(labels, np.float32), np.array(preds, np.float32), cold


def metric_value(name, label, prediction):
    """RegressionMetrics: rmse and mse from the L2 norm of the residuals (summed in row order), mae from the sum of
    their absolute values in row order; NaN for no rows."""
    d = [float(a) - float(b) for a, b in zip(np.asarray(label, np.float32), np.asarray(prediction, np.float32))]
    if not d:
        return float("nan")
    if name == "mae":
        s = 0.0
        for x in d:
            s += abs(x)
        return s / len(d)
    ss = 0.0
    for x in d:
        ss += x * x
    norm = math.sqrt(ss)
    return norm * norm / len(d) if name == "mse" else math.sqrt(norm * norm / len(d))


def java_compare(a, b):
    """java.lang.Double.compare for the metric values: NaN above everything, equal values equal."""
    if math.isnan(a) or math.isnan(b):
        return int(math.isnan(a)) - int(math.isnan(b))
    return (a > b) - (a < b)


def cross_validate(ratings, pairs, num_folds=10, metric="rmse", cold_start_strategy="nan", seed=0, rank=10,
                   max_iter=5, reg_param=0.01, als_seed=0, fit=X.fit):
    """CrossValidator.fit: returns dict(avg_metrics, fold_metrics [k][P], best_index, param_maps, cold_rows [k])."""
    n = len(ratings["userId"])
    fold = fold_of(n, num_folds, seed)
    points = [dict(dict(rank=rank, max_iter=max_iter, reg_param=reg_param), **pm) for pm in grid(pairs)]
    fold_metrics, cold_rows = [], []
    for f in range(num_folds):
        tr, va = fold != f, fold == f
        val = {c: np.asarray(v)[va] for c, v in ratings.items()}
        row = []
        for p in points:
            model = fit(np.asarray(ratings["userId"])[tr], np.asarray(ratings["movieId"])[tr],
                        np.asarray(ratings["rating"], np.float32)[tr], rank=p["rank"], max_iter=p["max_iter"],
                        reg_param=p["reg_param"], seed=als_seed)
            label, pred, cold = transform(model, val, cold_start_strategy)
            row.append(metric_value(metric, label, pred))
        cold_rows.append(cold)
        fold_metrics.append(row)
    avg = []
    for p in range(len(points)):
        s = 0.0
        for f in range(num_folds):
            s += fold_metrics[f][p]
        avg.append(s / num_folds)
    best = 0
    for i in range(1, len(avg)):
        if java_compare(avg[i], avg[best]) < 0:
            best = i
    return {"avg_metrics": avg, "fold_metrics": fold_metrics, "best_index": best, "param_maps": points,
            "cold_rows": cold_rows}
