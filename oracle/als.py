"""numpy restatement of the reference's CollaborativeFiltering job: Spark ML ALS (explicit feedback), its
`transform` with coldStartStrategy "drop", the RMSE and recommendForAll (DESIGN.md section 4.13).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT.  Spark's internals are restated from memory of Spark 2.4's
`ml/recommendation/ALS.scala` and the reference BLAS / LAPACK loops it calls through netlib-java's F2J fallback;
no ALS output of the reference is shipped, so parity with Spark is unpinned.  The work is vectorised across
entities, but every sum of one entity keeps the rule's order with one rounding per operation: numpy's pairwise
`sum` and BLAS `dot` are never used on those values.
"""
from __future__ import annotations

import math

import numpy as np

from .item2vec import splitmix

f32 = np.float32


class SingularError(ValueError):
    """A normal-equation system with a pivot <= 0 or NaN (Spark's SingularMatrixException)."""

    def __init__(self, side, entity_id, iteration):
        super().__init__("singular normal equations for %s %d in iteration %d" % (side, entity_id, iteration))
        self.side, self.entity_id, self.iteration = side, entity_id, iteration


def init_factor(seed, user_id, rank):
    """`rank` draws of nextGaussian's polar method on uniforms (splitmix(splitmix(seed, user_id), c) >> 11) / 2^53,
    each cast to float32, then scaled by 1.0f / snrm2 (reference BLAS's scaled sum of squares, in float)."""
    key = splitmix(seed & (2 ** 64 - 1), user_id)
    c = 0
    out = []
    while len(out) < rank:
        while True:
            v1 = 2 * ((splitmix(key, c) >> 11) * 2.0 ** -53) - 1
            v2 = 2 * ((splitmix(key, c + 1) >> 11) * 2.0 ** -53) - 1
            c += 2
            s = v1 * v1 + v2 * v2
            if s < 1 and s != 0:
                break
        m = math.sqrt(-2 * math.log(s) / s)
        out += [f32(v1 * m), f32(v2 * m)]
    x = np.array(out[:rank], np.float32)
    scale, ssq = f32(0), f32(1)
    for v in x:
        if v == 0:
            continue
        a = f32(abs(v))
        if scale < a:
            t = f32(scale / a)
            ssq = f32(f32(1) + f32(ssq * f32(t * t)))
            scale = a
        else:
            t = f32(a / scale)
            ssq = f32(ssq + f32(t * t))
    inv = f32(f32(1) / f32(scale * f32(np.sqrt(ssq))))
    return (x * inv).astype(np.float32)


def init_user_factors(user_ids, rank, seed):
    return np.stack([init_factor(seed, int(u), rank) for u in np.asarray(user_ids).tolist()]).astype(np.float32)


def layouts(user, movie, rating):
    """Dense ids and both layouts.  Returns (user ids, movie ids, by_movie, by_user); a layout is (off [nE + 1],
    src [n] counterpart dense index, r [n] float32 rating), each entity's ratings in ascending counterpart id with
    duplicates in input order."""
    user = np.asarray(user, np.int64)
    movie = np.asarray(movie, np.int64)
    r = np.asarray(rating, np.float32)
    uids, du = np.unique(user, return_inverse=True)
    mids, dm = np.unique(movie, return_inverse=True)
    idx = np.arange(len(user))

    def side(ent, cnt, nE):
        order = np.lexsort((idx, cnt, ent))
        off = np.r_[0, np.cumsum(np.bincount(ent, minlength=nE))].astype(np.int32)
        return off, cnt[order].astype(np.int32), r[order]

    return (uids.astype(np.int32), mids.astype(np.int32), side(dm, du, len(mids)), side(du, dm, len(uids)))


def solve_half(lay, srcF, k, reg):
    """One computeFactors: per entity NormalEquation (dspr / daxpy in rating order, double), lambda = n * reg on the
    diagonal, then dppsv "U".  Returns (dst float32 [nE][k], the first singular entity or -1)."""
    A, B = normal_equations(lay, srcF, k, reg)
    y, bad = cholesky_solve(A, B)
    first = int(np.flatnonzero(bad)[0]) if bad.any() else -1
    return y.astype(np.float32), first


def normal_equations(lay, srcF, k, reg):
    """Per entity ata + lambda I ([nE][k][k]: its upper triangle is the packed ata the solve reads) and atb [nE][k]."""
    off, src, r = lay
    nE = len(off) - 1
    cnt = np.diff(off)
    by_len = np.argsort(-cnt, kind="stable")               # the active entities are a prefix at each position
    A = np.zeros((nE, k, k))
    B = np.zeros((nE, k))
    scnt = cnt[by_len]
    start = off[:-1][by_len]
    srcD = srcF.astype(np.float64)
    for t in range(int(cnt.max()) if nE else 0):
        a = int(np.count_nonzero(scnt > t))                # entities with more than t ratings
        ents = by_len[:a]
        p = start[:a] + t
        X = srcD[src[p]]
        prod = X[:, :, None] * X[:, None, :]
        A[ents] = A[ents] + np.where(X[:, None, :] != 0, prod, 0.0)
        rv = r[p].astype(np.float64)[:, None]
        B[ents] = B[ents] + np.where(rv != 0, rv * X, 0.0)
    lam = cnt.astype(np.float64) * reg
    for j in range(k):
        A[:, j, j] = A[:, j, j] + lam
    return A, B


def cholesky_solve(A, B):
    """dppsv "U" on each entity's system: dpptrf, then dpptrs's two dtpsv.  Returns (x double [nE][k], singular
    [nE] bool: a pivot <= 0 or NaN)."""
    A, B = A.copy(), B.copy()
    nE, k = B.shape
    bad = np.zeros(nE, bool)
    with np.errstate(all="ignore"):
        for j in range(k):                                  # dpptrf "U"
            for jj in range(j):
                t = A[:, jj, j].copy()
                for i in range(jj):
                    t = t - A[:, i, jj] * A[:, i, j]
                A[:, jj, j] = t / A[:, jj, jj]
            dd = np.zeros(nE)
            for i in range(j):
                dd = dd + A[:, i, j] * A[:, i, j]
            ajj = A[:, j, j] - dd
            bad |= ~(ajj > 0)
            A[:, j, j] = np.sqrt(np.where(ajj > 0, ajj, 1.0))
        y = B
        for j in range(k):                                  # dtpsv "U", "T"
            t = y[:, j].copy()
            for i in range(j):
                t = t - A[:, i, j] * y[:, i]
            y[:, j] = t / A[:, j, j]
        for j in range(k - 1, -1, -1):                      # dtpsv "U", "N"
            nz = y[:, j] != 0
            yj = np.where(nz, y[:, j] / A[:, j, j], y[:, j])
            y[:, j] = yj
            for i in range(j):
                y[:, i] = np.where(nz, y[:, i] - yj * A[:, i, j], y[:, i])
    return y, bad


def fit(user, movie, rating, rank=10, max_iter=5, reg_param=0.01, seed=0, item_init=None, solver=solve_half,
        init=init_user_factors):
    """ALS.fit: returns (user ids, user factors, movie ids, movie factors).  `item_init`, Spark's initial item
    factors, is accepted and never read: each iteration solves the movies first."""
    uids, mids, by_movie, by_user = layouts(user, movie, rating)
    U = init(uids, rank, seed)
    M = np.zeros((len(mids), rank), np.float32) if item_init is None else np.asarray(item_init, np.float32)
    for it in range(1, max_iter + 1):
        for side, lay, ids in (("movie", by_movie, mids), ("user", by_user, uids)):
            out, bad = solver(lay, U if side == "movie" else M, rank, reg_param)
            if bad >= 0:
                raise SingularError(side, int(ids[bad]), it)
            if side == "movie":
                M = out
            else:
                U = out
    return uids, U, mids, M


def predict(uf, mf):
    """ALSModel's float dot, row by row: dot += u(d) * m(d) from 0.0f, d ascending."""
    s = np.zeros(uf.shape[0], np.float32)
    for d in range(uf.shape[1]):
        s = s + uf[:, d] * mf[:, d]
    return s


def recommend(src, dst_ids, dst, num):
    """recommendForAll: per source the min(num, n_dst) destinations of highest score (NaN as -inf), ties to the
    lower destination id (`dst_ids` ascending), best first.  Returns (ids int32, scores float32)."""
    src = np.asarray(src, np.float32)
    dst = np.asarray(dst, np.float32)
    S = np.zeros((src.shape[0], dst.shape[0]), np.float32)
    for d in range(src.shape[1]):
        S = S + src[:, d, None] * dst[None, :, d]
    key = np.where(np.isnan(S), -np.inf, S).astype(np.float64)
    L = min(int(num), dst.shape[0])
    order = np.argsort(-key, axis=1, kind="stable")[:, :L]
    return np.asarray(dst_ids, np.int32)[order], np.take_along_axis(S, order, axis=1)


def rmse(label, prediction):
    """RegressionEvaluator("rmse") as Spark 2.4's RegressionMetrics computes it: the squared norm of
    (label - prediction) in double, summed in row order, through sqrt then squared, over the count, then sqrt."""
    d = np.asarray(label, np.float32).astype(np.float64) - np.asarray(prediction, np.float32).astype(np.float64)
    ss = float(np.cumsum(d * d)[-1]) if d.size else 0.0
    n2 = math.sqrt(ss)
    return math.sqrt(n2 * n2 / d.size)
