"""Collaborative filtering on the GPU: ALS factors, test RMSE and top-k recommendations.

This is the reference's Spark job `OFF/model/CollaborativeFiltering.scala` (and its PySpark twin): split ratings.csv
0.8 / 0.2, train Spark ML's `ALS` (explicit feedback, maxIter 5, regParam 0.01, rank 10) on the first part, take
the RMSE of `transform` on the second with coldStartStrategy "drop", and recommend 10 movies per user and 10 users
per movie.  DESIGN.md section 4.13 gives the semantics and the orders Spark leaves open; `oracle/als.py` restates
them.

* `random_split` is `Dataset.randomSplit` with a counter-based uniform per row.
* `als` trains on one device (`srs_als_fit_host`) and returns an `AlsModel`.
* `AlsModel.transform` predicts on the host with ALSModel's float dot; `rmse` is RegressionEvaluator("rmse").
* `AlsModel.recommend_for_*` score and keep the top `num` on one device (`srs_als_recommend_host`).

    python -m sparrowrecsys_b200.collab ratings.csv
"""
from __future__ import annotations

import ctypes as C
import math
import sys
from typing import Mapping, Sequence, Tuple

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

    def transform(self, ratings: Mapping[str, np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
        """ALSModel.transform with coldStartStrategy "drop": rows whose user or movie has no factor are dropped.
        Returns (kept row indices int64, predictions float32): dot += u(d) * m(d) from 0.0f, d ascending."""
        user = np.asarray(ratings["userId"], np.int64)
        movie = np.asarray(ratings["movieId"], np.int64)
        ui = np.searchsorted(self.user_ids, user)
        mi = np.searchsorted(self.item_ids, movie)
        ok = (ui < len(self.user_ids)) & (mi < len(self.item_ids))
        ok[ok] &= (self.user_ids[ui[ok]] == user[ok]) & (self.item_ids[mi[ok]] == movie[ok])
        rows = np.flatnonzero(ok)
        uf, mf = self.user_factors[ui[rows]], self.item_factors[mi[rows]]
        pred = np.zeros(len(rows), np.float32)
        for d in range(self.rank):
            pred = pred + uf[:, d] * mf[:, d]
        return rows, pred

    def recommend_for_all_users(self, num: int):
        """(user ids [U], movie ids [U][L], scores [U][L]), L = min(num, movies)."""
        ids, sc = recommend(self.user_factors, self.item_ids, self.item_factors, num, self.device)
        return self.user_ids, ids, sc

    def recommend_for_all_items(self, num: int):
        """(movie ids [M], user ids [M][L], scores [M][L]), L = min(num, users)."""
        ids, sc = recommend(self.item_factors, self.user_ids, self.user_factors, num, self.device)
        return self.item_ids, ids, sc

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
        seed: int = 0, device: int = 0) -> AlsModel:
    """ALS.fit (explicit feedback) on `ratings` (userId, movieId, rating; as `featureeng.load_ratings_csv` returns)
    on `device`.  Ratings are cast to float32 as Spark casts its rating column.  The same inputs give the same
    bits."""
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
    _lib.check(_lib.load().srs_als_fit_host(_p(user), _p(movie), _p(rating), n, C.byref(params), device, cu, cm,
                                            _p(uids), _p(uf), C.byref(nu), _p(mids), _p(mf), C.byref(nm)))
    return AlsModel(uids[:nu.value].copy(), uf[:nu.value].copy(), mids[:nm.value].copy(), mf[:nm.value].copy(),
                    device)


def rmse(labels, predictions) -> float:
    """RegressionEvaluator("rmse") as Spark 2.4's RegressionMetrics computes it: the L2 norm of (label -
    prediction) in double, summed in row order, squared, over the count, then the square root."""
    d = np.asarray(labels, np.float32).astype(np.float64) - np.asarray(predictions, np.float32).astype(np.float64)
    if d.size == 0:
        return float("nan")
    norm = math.sqrt(float(np.cumsum(d * d)[-1]))
    return math.sqrt(norm * norm / d.size)


def _show(title, ids, rec, sc, rows=10):
    print(title)
    for i in range(min(rows, len(ids))):
        print("%d\t[%s]" % (ids[i], ", ".join("[%d, %s]" % (a, repr(float(b))) for a, b in zip(rec[i], sc[i]))))


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) != 1:
        sys.stderr.write("usage: python -m sparrowrecsys_b200.collab ratings.csv\n")
        return 2
    from .featureeng import load_ratings_csv
    r = load_ratings_csv(argv[0])
    train_rows, test_rows = random_split(len(r["userId"]), (0.8, 0.2), seed=0)
    train = {k: v[train_rows] for k, v in r.items()}
    test = {k: v[test_rows] for k, v in r.items()}
    model = als(train, rank=10, max_iter=5, reg_param=0.01, seed=0)
    for name, ids, f in (("itemFactors", model.item_ids, model.item_factors),
                         ("userFactors", model.user_ids, model.user_factors)):
        print(name)
        for i in range(min(10, len(ids))):
            print("%d\t[%s]" % (ids[i], ", ".join(repr(float(v)) for v in f[i])))
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
    return 0


if __name__ == "__main__":
    sys.exit(main())
