"""Collaborative filtering on the GPU: ALS factors (explicit or implicit feedback), test RMSE or ranking metrics,
and top-k recommendations.

This is the reference's Spark job `OFF/model/CollaborativeFiltering.scala` (and its PySpark twin): split ratings.csv
0.8 / 0.2, train Spark ML's `ALS` (explicit feedback, maxIter 5, regParam 0.01, rank 10) on the first part, take
the RMSE of `transform` on the second with coldStartStrategy "drop", and recommend 10 movies per user and 10 users
per movie.  DESIGN.md section 4.13 gives the semantics and the orders Spark leaves open; `oracle/als.py` restates
them.

* `random_split` is `Dataset.randomSplit` with a counter-based uniform per row.
* `als` trains on one device (`srs_als_fit_host`) and returns an `AlsModel`.
* `AlsModel.transform` predicts on the host with ALSModel's float dot; `rmse` is RegressionEvaluator("rmse").
* `AlsModel.recommend_for_*` score and keep the top `num` on one device (`srs_als_recommend_host`).
* `cross_validate` is the job's last step, `CrossValidator` over a `ParamGridBuilder` grid: every fold x grid model
  trained in one batched device pass (`als_folds`, `srs_als_fit_folds_host`; DESIGN.md section 4.15).
* `als(..., implicit_prefs=True, alpha=...)` is the estimator's implicit-feedback mode (`srs_als_fit_implicit_host`),
  and `ranking_metrics` / `AlsModel.ranking_metrics` are mllib's `RankingMetrics` - precision@k, NDCG@k and MAP -
  with the per-query values on the device (`srs_ranking_metrics_host`; DESIGN.md section 4.17).
* `als(..., nonnegative=True)` is the estimator's `nonnegative` mode: every factor solved under x >= 0 by Spark's
  NNLSSolver, explicit or implicit (`srs_als_fit_nonnegative_host`), and a model mapping of `als_folds` /
  `cross_validate`'s grid may set "nonnegative" (`srs_als_fit_folds_nonnegative_host`; DESIGN.md section 4.21).

    python -m sparrowrecsys_b200.collab ratings.csv [--nonnegative] [--cv | --implicit [--alpha A]]
"""
from __future__ import annotations

import ctypes as C
import math
import struct
import sys
from dataclasses import dataclass
from typing import List, Mapping, Sequence, Tuple

import numpy as np

from . import _lib

_M64 = (1 << 64) - 1


def _uniforms(seed: int, n: int) -> np.ndarray:
    """Row i's uniform in [0, 1): the top 53 bits of splitmix(seed, i) over 2^53 (srs_fill_uniform's hash)."""
    i = np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(seed & _M64) + (i + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def random_split(n: int, weights: Sequence[float] = (0.8, 0.2), seed: int = 0):
    """Dataset.randomSplit(weights): row i goes to part j when lb_j <= u_i < ub_j, the bounds being the running sums
    of the weights over their total (Spark's normalised cumulative weights).  Returns one int64 index array per part,
    ascending."""
    w = [float(x) for x in weights]
    if not w or any(not math.isfinite(x) or x < 0 for x in w) or sum(w) <= 0:
        raise ValueError("weights must be finite, non-negative and not all zero")
    total = sum(w)
    bounds = [0.0]
    for x in w:
        bounds.append(bounds[-1] + x / total)
    u = _uniforms(int(seed), int(n))
    return [np.flatnonzero((u >= lo) & (u < hi)) for lo, hi in zip(bounds[:-1], bounds[1:])]


def _p(a):
    return a.ctypes.data


def recommend(src_factors, dst_ids, dst_factors, num: int, device: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """recommendForAll's scoring on the device: per source row the min(num, n_dst) destinations of highest float
    dot, best first, ties to the lower destination id (`dst_ids` strictly ascending).  Returns (ids int32, scores
    float32), both [n_src][min(num, n_dst)]."""
    src = np.ascontiguousarray(src_factors, np.float32)
    dst = np.ascontiguousarray(dst_factors, np.float32)
    ids = np.ascontiguousarray(dst_ids, np.int32)
    if src.ndim != 2 or dst.ndim != 2 or src.shape[1] != dst.shape[1] or ids.shape != (dst.shape[0],):
        raise ValueError("src [n, rank], dst_ids [m] and dst [m, rank] expected")
    L = min(int(num), dst.shape[0])
    out_i = np.zeros((src.shape[0], max(L, 0)), np.int32)
    out_s = np.zeros((src.shape[0], max(L, 0)), np.float32)
    _lib.check(_lib.load().srs_als_recommend_host(_p(src), src.shape[0], _p(ids), _p(dst), dst.shape[0],
                                                  src.shape[1], int(num), device, _p(out_i), _p(out_s)))
    return out_i, out_s


class AlsModel:
    """ALSModel: user and movie factors by ascending id."""

    def __init__(self, user_ids, user_factors, item_ids, item_factors, device: int = 0):
        self.user_ids, self.user_factors = user_ids, user_factors
        self.item_ids, self.item_factors = item_ids, item_factors
        self.rank = user_factors.shape[1]
        self.device = device

    def _lookup(self, ratings):
        """(user factor row, movie factor row, both known) of each rating row."""
        user = np.asarray(ratings["userId"], np.int64)
        movie = np.asarray(ratings["movieId"], np.int64)
        ui = np.searchsorted(self.user_ids, user)
        mi = np.searchsorted(self.item_ids, movie)
        ok = (ui < len(self.user_ids)) & (mi < len(self.item_ids))
        ok[ok] &= (self.user_ids[ui[ok]] == user[ok]) & (self.item_ids[mi[ok]] == movie[ok])
        return ui, mi, ok

    def cold_rows(self, ratings: Mapping[str, np.ndarray]) -> int:
        """The number of rows whose user or movie has no factor."""
        return int(np.count_nonzero(~self._lookup(ratings)[2]))

    def transform(self, ratings: Mapping[str, np.ndarray],
                  cold_start_strategy: str = "drop") -> Tuple[np.ndarray, np.ndarray]:
        """ALSModel.transform: dot += u(d) * m(d) from 0.0f, d ascending, for rows whose user and movie have
        factors.  coldStartStrategy "drop" drops the other rows; "nan" (Spark's default) keeps them with a NaN
        prediction.  Returns (row indices int64, predictions float32)."""
        if cold_start_strategy not in ("drop", "nan"):
            raise ValueError("cold_start_strategy must be 'drop' or 'nan', not %r" % (cold_start_strategy,))
        ui, mi, ok = self._lookup(ratings)
        rows = np.flatnonzero(ok)
        uf, mf = self.user_factors[ui[rows]], self.item_factors[mi[rows]]
        pred = np.zeros(len(rows), np.float32)
        for d in range(self.rank):
            pred = pred + uf[:, d] * mf[:, d]
        if cold_start_strategy == "drop":
            return rows, pred
        out = np.full(len(ok), np.nan, np.float32)
        out[rows] = pred
        return np.arange(len(ok), dtype=np.int64), out

    def recommend_for_all_users(self, num: int):
        """(user ids [U], movie ids [U][L], scores [U][L]), L = min(num, movies)."""
        ids, sc = recommend(self.user_factors, self.item_ids, self.item_factors, num, self.device)
        return self.user_ids, ids, sc

    def recommend_for_all_items(self, num: int):
        """(movie ids [M], user ids [M][L], scores [M][L]), L = min(num, users)."""
        ids, sc = recommend(self.item_factors, self.user_ids, self.user_factors, num, self.device)
        return self.item_ids, ids, sc

    def ranking_queries(self, ratings: Mapping[str, np.ndarray], threshold: float = 0.0):
        """The queries of `ranking_metrics`: (the users of `ratings` that have factors, ascending; their rows in
        user_factors; a CSR tuple (offsets, movie ids) of each one's movies rated above `threshold`)."""
        user = np.asarray(ratings["userId"], np.int64)
        movie = np.asarray(ratings["movieId"], np.int64)
        rel = np.asarray(ratings["rating"], np.float32) > np.float32(threshold)
        at = self._subset(user, self.user_ids)
        order = np.lexsort((movie, user))
        user, movie = user[order][rel[order]], movie[order][rel[order]]
        users = self.user_ids[at].astype(np.int64)
        lo = np.searchsorted(user, users, "left")
        hi = np.searchsorted(user, users, "right")
        off = np.zeros(len(users) + 1, np.int32)
        off[1:] = np.cumsum(hi - lo)
        ids = np.concatenate([movie[a:b] for a, b in zip(lo, hi)]) if len(users) else np.zeros(0)
        return self.user_ids[at], at, (off, ids.astype(np.int32))

    def ranking_metrics(self, ratings: Mapping[str, np.ndarray], k: int, threshold: float = 0.0) -> dict:
        """RankingMetrics of recommend_for_user_subset(users, k) against held-out `ratings` (Spark 2.4 has no
        ranking evaluator for ALS; this is how its users score implicit models): the queries are the users of
        `ratings` that have factors, ascending; each one's relevant items are its movies rated above `threshold`
        (preference [rating > 0] by default; a movie without a factor stays relevant and is never recommended).  A
        user with none scores 0 and still counts.  Returns `ranking_metrics`' dict."""
        users, _, labels = self.ranking_queries(ratings, threshold)
        _, pred, _ = self.recommend_for_user_subset(users, k)
        return ranking_metrics(pred, labels, k, self.device)

    @staticmethod
    def _subset(ids, known):
        q = np.unique(np.asarray(ids, np.int64))
        at = np.searchsorted(known, q)
        hit = at < len(known)
        hit[hit] &= known[at[hit]] == q[hit]
        return at[hit]

    def recommend_for_user_subset(self, user_ids, num: int):
        """recommendForUserSubset: the distinct given users that have factors, ascending, as recommend_for_all_users."""
        at = self._subset(user_ids, self.user_ids)
        ids, sc = recommend(self.user_factors[at], self.item_ids, self.item_factors, num, self.device)
        return self.user_ids[at], ids, sc

    def recommend_for_item_subset(self, item_ids, num: int):
        """recommendForItemSubset: the distinct given movies that have factors, ascending."""
        at = self._subset(item_ids, self.item_ids)
        ids, sc = recommend(self.item_factors[at], self.user_ids, self.user_factors, num, self.device)
        return self.item_ids[at], ids, sc


def als(ratings: Mapping[str, np.ndarray], rank: int = 10, max_iter: int = 5, reg_param: float = 0.01,
        seed: int = 0, device: int = 0, implicit_prefs: bool = False, alpha: float = 1.0,
        nonnegative: bool = False) -> AlsModel:
    """ALS.fit on `ratings` (userId, movieId, rating; as `featureeng.load_ratings_csv` returns) on `device`:
    explicit feedback, or with `implicit_prefs` the implicit mode with confidence 1 + alpha |rating| and
    preference [rating > 0] (DESIGN.md section 4.17).  With `nonnegative` every factor is solved under x >= 0 by
    Spark's NNLSSolver (DESIGN.md section 4.21).  Ratings are cast to float32 as Spark casts its rating column.  The
    same inputs give the same bits."""
    user = np.ascontiguousarray(ratings["userId"], np.int32)
    movie = np.ascontiguousarray(ratings["movieId"], np.int32)
    rating = np.ascontiguousarray(ratings["rating"], np.float32)
    n = user.shape[0]
    if movie.shape[0] != n or rating.shape[0] != n:
        raise ValueError("ratings columns differ in length")
    cu, cm = max(1, int(np.unique(user).size)), max(1, int(np.unique(movie).size))
    k = int(rank)
    uids, uf = np.zeros(cu, np.int32), np.zeros((cu, max(k, 1)), np.float32)
    mids, mf = np.zeros(cm, np.int32), np.zeros((cm, max(k, 1)), np.float32)
    params = _lib.SrsAlsParams(k, int(max_iter), float(reg_param), int(seed) & _M64)
    nu, nm = C.c_int32(0), C.c_int32(0)
    args = (_p(user), _p(movie), _p(rating), n, C.byref(params), device, cu, cm, _p(uids), _p(uf), C.byref(nu),
            _p(mids), _p(mf), C.byref(nm))
    if nonnegative:
        _lib.check(_lib.load().srs_als_fit_nonnegative_host(*args, int(bool(implicit_prefs)), float(alpha)))
    elif implicit_prefs:
        _lib.check(_lib.load().srs_als_fit_implicit_host(*args, float(alpha)))
    else:
        _lib.check(_lib.load().srs_als_fit_host(*args))
    return AlsModel(uids[:nu.value].copy(), uf[:nu.value].copy(), mids[:nm.value].copy(), mf[:nm.value].copy(),
                    device)


def ranking_metrics(pred_ids, labels, k: int, device: int = 0) -> dict:
    """mllib RankingMetrics (Spark 2.4) on the device: `pred_ids` [n][L] best first, `labels` the relevant ids of
    each query - a list of n sequences, or a CSR tuple (offsets [n + 1], ids) - taken as sets.  Returns
    precision_at_k (hits in the first min(L, k) over k), ndcg_at_k and mean_average_precision (over the whole
    list, as Spark 2.4's is), each StatCounter's mean over the queries in order; an empty label set scores 0."""
    pred = np.ascontiguousarray(pred_ids, np.int32)
    if pred.ndim == 1 and pred.size == 0:
        pred = pred.reshape(0, 0)
    if pred.ndim != 2:
        raise ValueError("pred_ids must be [n_queries][L]")
    if isinstance(labels, tuple):
        off, ids = (np.ascontiguousarray(x, np.int32) for x in labels)
        if off.shape != (pred.shape[0] + 1,) or ids.ndim != 1 or (len(off) and (off[0] != 0 or off[-1] != len(ids))):
            raise ValueError("CSR labels need offsets [n + 1] from 0 to len(ids)")
    else:
        if len(labels) != pred.shape[0]:
            raise ValueError("%d label sets for %d queries" % (len(labels), pred.shape[0]))
        sizes = [len(x) for x in labels]
        off = np.zeros(len(sizes) + 1, np.int32)
        off[1:] = np.cumsum(sizes)
        ids = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int64) for x in labels]) if sizes
                                   else np.zeros(0), np.int32)
    means = np.zeros(3)
    _lib.check(_lib.load().srs_ranking_metrics_host(_p(pred), pred.shape[0], pred.shape[1], _p(off),
                                                    _p(ids if ids.size else np.zeros(1, np.int32)), int(k), device,
                                                    None, _p(means)))
    return {"precision_at_k": float(means[0]), "ndcg_at_k": float(means[1]),
            "mean_average_precision": float(means[2])}


MAX_BATCH_MODELS = 64


def als_folds(ratings: Mapping[str, np.ndarray], fold, n_folds: int, models: Sequence[Mapping], seed: int = 0,
              device: int = 0) -> List[AlsModel]:
    """Many ALS.fit calls over one rating set in one device pass (`srs_als_fit_folds_host`).  `fold` [n] gives each
    row a fold in 0..n_folds-1; each of the (at most 64) `models` is a mapping with rank, max_iter, reg_param and
    exclude_fold (-1: train on every row), and optionally nonnegative (default False).  Model m trains on the rows
    outside its excluded fold, and its factors are bit for bit `als` on those rows in input order with its settings
    and `seed`."""
    user = np.ascontiguousarray(ratings["userId"], np.int32)
    movie = np.ascontiguousarray(ratings["movieId"], np.int32)
    rating = np.ascontiguousarray(ratings["rating"], np.float32)
    fold = np.ascontiguousarray(fold, np.int32)
    n = user.shape[0]
    if movie.shape[0] != n or rating.shape[0] != n or fold.shape[0] != n:
        raise ValueError("ratings columns and fold differ in length")
    M = len(models)
    specs = (_lib.SrsAlsModel * max(M, 1))()
    for i, p in enumerate(models):
        specs[i] = _lib.SrsAlsModel(int(p["rank"]), int(p["max_iter"]), float(p["reg_param"]),
                                    int(p["exclude_fold"]))
    cu, cm = max(1, int(np.unique(user).size)), max(1, int(np.unique(movie).size))
    ranks = [max(1, int(p["rank"])) for p in models] or [1]
    uids, mids = np.zeros((len(ranks), cu), np.int32), np.zeros((len(ranks), cm), np.int32)
    uf, mf = np.zeros(cu * sum(ranks), np.float32), np.zeros(cm * sum(ranks), np.float32)
    nu, nm = np.zeros(len(ranks), np.int32), np.zeros(len(ranks), np.int32)
    args = (_p(user), _p(movie), _p(rating), _p(fold), n, int(n_folds), specs, M, int(seed) & _M64, device, cu, cm,
            _p(uids), _p(uf), _p(nu), _p(mids), _p(mf), _p(nm))
    nonneg = np.array([int(bool(p.get("nonnegative", False))) for p in models] or [0], np.int32)
    if nonneg.any():
        _lib.check(_lib.load().srs_als_fit_folds_nonnegative_host(*args, _p(nonneg)))
    else:
        _lib.check(_lib.load().srs_als_fit_folds_host(*args))
    out, r0 = [], 0
    for m, k in enumerate(ranks[:M]):
        U = uf[cu * r0:cu * (r0 + k)].reshape(cu, k)
        V = mf[cm * r0:cm * (r0 + k)].reshape(cm, k)
        out.append(AlsModel(uids[m, :nu[m]].copy(), U[:nu[m]].copy(), mids[m, :nm[m]].copy(), V[:nm[m]].copy(),
                            device))
        r0 += k
    return out


def _sum_sq(labels, predictions):
    d = np.asarray(labels, np.float32).astype(np.float64) - np.asarray(predictions, np.float32).astype(np.float64)
    return d, (float(np.cumsum(d * d)[-1]) if d.size else 0.0)


def rmse(labels, predictions) -> float:
    """RegressionEvaluator("rmse") as Spark 2.4's RegressionMetrics computes it: the L2 norm of (label -
    prediction) in double, summed in row order, squared, over the count, then the square root."""
    d, ss = _sum_sq(labels, predictions)
    if d.size == 0:
        return float("nan")
    norm = math.sqrt(ss)
    return math.sqrt(norm * norm / d.size)


def mse(labels, predictions) -> float:
    """RegressionEvaluator("mse"): rmse's value before the square root, the squared L2 norm over the count."""
    d, ss = _sum_sq(labels, predictions)
    if d.size == 0:
        return float("nan")
    norm = math.sqrt(ss)
    return norm * norm / d.size


def mae(labels, predictions) -> float:
    """RegressionEvaluator("mae"): |label - prediction| in double, summed in row order, over the count."""
    d, _ = _sum_sq(labels, predictions)
    if d.size == 0:
        return float("nan")
    return float(np.cumsum(np.abs(d))[-1]) / d.size


METRICS = {"rmse": rmse, "mse": mse, "mae": mae}
_GRID_PARAMS = ("rank", "reg_param", "max_iter", "nonnegative")


def fold_ids(n: int, num_folds: int, seed: int = 0) -> np.ndarray:
    """MLUtils.kFold's fold of each row (0-based): row i draws `_uniforms(seed, n)[i]` once, the same draw for every
    fold, and fold f validates the rows with lb <= u < ub, lb = (f - 1) / k and ub = f / k (f = 1..k) computed as
    float32 quotients (Spark's `(fold - 1) / numFolds.toFloat`) and widened to double.  Returns int32 [n]."""
    if int(num_folds) < 2:
        raise ValueError("num_folds must be >= 2, not %d" % int(num_folds))
    return _fold_of(_uniforms(int(seed), int(n)), int(num_folds))


def _fold_of(u, k):
    out = np.full(len(u), -1, np.int32)
    for f in range(1, k + 1):
        lb = float(np.float32(f - 1) / np.float32(k))
        ub = float(np.float32(f) / np.float32(k))
        out[(u >= lb) & (u < ub)] = f - 1
    return out


def k_fold(n: int, num_folds: int, seed: int = 0):
    """MLUtils.kFold: one (training rows, validation rows) pair of ascending int64 indices per fold, the training
    rows the complement of the validation rows (see `fold_ids`)."""
    f = fold_ids(n, num_folds, seed)
    return [(np.flatnonzero(f != i), np.flatnonzero(f == i)) for i in range(int(num_folds))]


def param_maps(param_grid) -> List[dict]:
    """ParamGridBuilder.build over an ordered list of (param, values) pairs (or a dict, in its order) of "rank",
    "reg_param", "max_iter" and "nonnegative": every combination, the first param varying fastest.  No params give one empty
    map, as Spark's builder does; a param with no values gives none, which is an error here."""
    pairs = list(param_grid.items()) if isinstance(param_grid, Mapping) else [tuple(p) for p in param_grid]
    names = [p[0] for p in pairs]
    if any(name not in _GRID_PARAMS for name in names) or len(set(names)) != len(names):
        raise ValueError("grid params must be distinct names from %s, not %s" % (_GRID_PARAMS, names))
    maps = [{}]
    for name, values in pairs:
        maps = [dict(m, **{name: v}) for v in values for m in maps]
    if not maps:
        raise ValueError("the parameter grid is empty")
    return maps


def _java_compare(a: float, b: float) -> int:
    """java.lang.Double.compare: numeric order, then the bits (-0.0 < 0.0, NaN above everything)."""
    if a < b:
        return -1
    if a > b:
        return 1

    def bits(x):
        return 0x7FF8000000000000 if math.isnan(x) else struct.unpack("<q", struct.pack("<d", x))[0]
    return (bits(a) > bits(b)) - (bits(a) < bits(b))


def average_metrics(fold_metrics) -> List[float]:
    """CrossValidator's avgMetrics from fold_metrics [k][P]: per grid point the sum over folds in fold order, in
    double from 0.0, over k."""
    k = len(fold_metrics)
    avg = []
    for p in range(len(fold_metrics[0])):
        s = 0.0
        for f in range(k):
            s += float(fold_metrics[f][p])
        avg.append(s / k)
    return avg


def best_index(metrics: Sequence[float]) -> int:
    """CrossValidator's minBy over the average metrics (rmse, mse and mae are smaller-is-better) in
    java.lang.Double.compare's order: NaN ranks last, and the first index wins a tie."""
    best = 0
    for i in range(1, len(metrics)):
        if _java_compare(float(metrics[i]), float(metrics[best])) < 0:
            best = i
    return best


@dataclass
class CrossValidation:
    """What `cross_validate` returns.  avg_metrics [P] and fold_metrics [k][P] follow param_maps' order;
    param_maps holds each grid point's full settings; cold_rows [k] counts each fold's validation rows whose user or
    movie has no factor in that fold's models."""
    avg_metrics: List[float]
    fold_metrics: List[List[float]]
    best_index: int
    best_params: dict
    best_model: AlsModel
    param_maps: List[dict]
    cold_rows: List[int]


def cross_validate(ratings: Mapping[str, np.ndarray], param_grid, num_folds: int = 10, metric: str = "rmse",
                   cold_start_strategy: str = "nan", seed: int = 0, rank: int = 10, max_iter: int = 5,
                   reg_param: float = 0.01, als_seed: int = 0, device: int = 0,
                   nonnegative: bool = False) -> CrossValidation:
    """CrossValidator(ALS, RegressionEvaluator(metric), param_grid, num_folds).fit(ratings) on the device.  Every
    fold x grid model is trained in batched passes of at most 64 models (`als_folds`); params not in the grid take
    rank, max_iter, reg_param and nonnegative, and every fit uses `als_seed`.  Each model predicts its validation rows with
    `cold_start_strategy` ("nan", the estimator's default, makes a fold with a cold row score NaN), avg_metrics[p]
    is the fold-order sum over k, and the best point (`best_index`) is refit on all rows by `als`."""
    if metric not in METRICS:
        raise ValueError("metric must be one of %s, not %r" % (sorted(METRICS), metric))
    if cold_start_strategy not in ("drop", "nan"):
        raise ValueError("cold_start_strategy must be 'drop' or 'nan', not %r" % (cold_start_strategy,))
    base = dict(rank=rank, max_iter=max_iter, reg_param=reg_param)
    if nonnegative:                                         # a call that never mentions it keeps today's maps
        base["nonnegative"] = True
    points = [dict(base, **pm) for pm in param_maps(param_grid)]
    k, P = int(num_folds), len(points)
    n = len(ratings["userId"])
    fold = fold_ids(n, k, seed)
    specs = [dict(p, exclude_fold=f) for f in range(k) for p in points]
    models = []
    for i in range(0, len(specs), MAX_BATCH_MODELS):
        models += als_folds(ratings, fold, k, specs[i:i + MAX_BATCH_MODELS], als_seed, device)
    fold_metrics, cold = [], []
    for f in range(k):
        val = {c: np.asarray(v)[fold == f] for c, v in ratings.items()}
        cold.append(models[f * P].cold_rows(val))
        row = []
        for p in range(P):
            rows, pred = models[f * P + p].transform(val, cold_start_strategy)
            row.append(METRICS[metric](np.asarray(val["rating"])[rows], pred))
        fold_metrics.append(row)
    avg = average_metrics(fold_metrics)
    best = best_index(avg)
    model = als(ratings, points[best]["rank"], points[best]["max_iter"], points[best]["reg_param"], als_seed, device,
                nonnegative=bool(points[best].get("nonnegative", False)))
    return CrossValidation(avg, fold_metrics, best, dict(points[best]), model, points, cold)


def _show(title, ids, rec, sc, rows=10):
    print(title)
    for i in range(min(rows, len(ids))):
        print("%d\t[%s]" % (ids[i], ", ".join("[%d, %s]" % (a, repr(float(b))) for a, b in zip(rec[i], sc[i]))))


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    usage = ("usage: python -m sparrowrecsys_b200.collab ratings.csv [--nonnegative] "
             "[--cv | --implicit [--alpha A]]\n")
    alpha = 1.0
    if "--alpha" in argv:
        at = argv.index("--alpha")
        try:
            alpha = float(argv[at + 1])
        except (IndexError, ValueError):
            sys.stderr.write(usage)
            return 2
        del argv[at:at + 2]
        if "--implicit" not in argv:
            sys.stderr.write(usage)
            return 2
    cv, implicit, nonneg = "--cv" in argv, "--implicit" in argv, "--nonnegative" in argv
    args = [a for a in argv if a not in ("--cv", "--implicit", "--nonnegative")]
    if len(args) != 1 or (cv and implicit):                 # CrossValidator has no ranking evaluator
        sys.stderr.write(usage)
        return 2
    from .featureeng import load_ratings_csv
    r = load_ratings_csv(args[0])
    train_rows, test_rows = random_split(len(r["userId"]), (0.8, 0.2), seed=0)
    train = {k: v[train_rows] for k, v in r.items()}
    test = {k: v[test_rows] for k, v in r.items()}
    model = als(train, rank=10, max_iter=5, reg_param=0.01, seed=0, implicit_prefs=implicit, alpha=alpha,
                nonnegative=nonneg)
    for name, ids, f in (("itemFactors", model.item_ids, model.item_factors),
                         ("userFactors", model.user_ids, model.user_factors)):
        print(name)
        for i in range(min(10, len(ids))):
            print("%d\t[%s]" % (ids[i], ", ".join(repr(float(v)) for v in f[i])))
    if implicit:                                            # preferences, not ratings: rank the held-out items
        m = model.ranking_metrics(test, 10)
        print("precisionAt(10) = %r" % m["precision_at_k"])
        print("ndcgAt(10) = %r" % m["ndcg_at_k"])
        print("meanAveragePrecision = %r" % m["mean_average_precision"])
    else:
        kept, pred = model.transform(test)
        print("Root-mean-square error = %r" % rmse(test["rating"][kept], pred))
    _show("userRecs", *model.recommend_for_all_users(10))
    _show("movieRecs", *model.recommend_for_all_items(10))
    _, first_users = np.unique(r["userId"], return_index=True)
    _, first_movies = np.unique(r["movieId"], return_index=True)
    users = r["userId"][np.sort(first_users)[:3]]          # distinct().limit(3): the first three seen
    movies = r["movieId"][np.sort(first_movies)[:3]]
    _show("userSubsetRecs", *model.recommend_for_user_subset(users, 10))
    _show("movieSubSetRecs", *model.recommend_for_item_subset(movies, 10))
    if cv:                                                  # cv.fit(test): regParam grid [0.01], 10 folds
        res = cross_validate(test, [("reg_param", [0.01])], num_folds=10, nonnegative=nonneg)
        print("avgMetrics = %r" % res.avg_metrics)
        print("cold validation rows per fold = %r" % res.cold_rows)
    return 0


if __name__ == "__main__":
    sys.exit(main())
