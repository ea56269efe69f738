"""numpy restatement of Spark ML ALS with implicitPrefs and of mllib's RankingMetrics (DESIGN.md section 4.17).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT.  Like oracle/als.py, which it builds on (layouts, init, the Cholesky
solve), it restates Spark 2.4's `ml/recommendation/ALS.scala` (`computeFactors`, `computeYtY`, `NormalEquation`)
and `mllib/evaluation/RankingMetrics.scala` from memory; parity with Spark is unpinned.  Every sum of one entity,
one YtY block or one query keeps the rule's order with one rounding per operation.
"""
from __future__ import annotations

import math

import numpy as np

from . import als as A

BLOCKS = 10                                                 # Spark's default numUserBlocks / numItemBlocks


def yty_blocks(ids):
    """Spark's ten blocks of YtY's summands: the dense indices of the entities with raw id mod 10 == b, ascending."""
    ids = np.asarray(ids, np.int64)
    return [np.flatnonzero(ids % BLOCKS == b) for b in range(BLOCKS)]


def yty(ids, srcF, order=tuple(range(BLOCKS))):
    """computeYtY: per block, NormalEquation.add(y, 0.0) - dspr("U", k, 1.0, y, ap), skipped for y(j) == 0 - over
    its entities in ascending id, from zero in double; then the blocks merged in `order` (daxpy(1.0) from zero).
    Returns the full [k][k] matrix whose upper triangle is the packed YtY."""
    X = np.asarray(srcF, np.float32).astype(np.float64)
    k = X.shape[1]
    members = yty_blocks(ids)
    part = np.zeros((BLOCKS, k, k))
    for t in range(max(len(m) for m in members)):
        live = [b for b in range(BLOCKS) if t < len(members[b])]
        x = X[[members[b][t] for b in live]]
        part[live] = part[live] + np.where(x[:, None, :] != 0, x[:, :, None] * x[:, None, :], 0.0)
    out = np.zeros((k, k))
    for b in order:
        out = out + part[b]
    return out


def normal_equations(lay, srcF, src_ids, k, reg, alpha):
    """Per entity (YtY + sum c1 y y^T + lambda I) [nE][k][k] (upper triangle as packed) and sum_{r > 0} (1 + c1) y
    [nE][k], with c1 = alpha |r| and lambda = reg * (its ratings > 0)."""
    off, src, r = lay
    nE = len(off) - 1
    cnt = np.diff(off)
    by_len = np.argsort(-cnt, kind="stable")
    A_ = np.broadcast_to(yty(src_ids, srcF), (nE, k, k)).copy()
    B = np.zeros((nE, k))
    scnt = cnt[by_len]
    start = off[:-1][by_len]
    srcD = np.asarray(srcF, np.float32).astype(np.float64)
    rr = np.asarray(r, np.float32)
    for t in range(int(cnt.max()) if nE else 0):
        a = int(np.count_nonzero(scnt > t))
        ents = by_len[:a]
        p = start[:a] + t
        X = srcD[src[p]]
        rv = rr[p].astype(np.float64)
        c1 = alpha * np.abs(rv)
        temp = c1[:, None] * X                              # dspr's temp = alpha * x(j)
        prod = X[:, :, None] * temp[:, None, :]
        keep = (c1[:, None, None] != 0) & (X[:, None, :] != 0)
        A_[ents] = A_[ents] + np.where(keep, prod, 0.0)
        b = 1.0 + c1
        B[ents] = B[ents] + np.where((rv > 0)[:, None], b[:, None] * X, 0.0)
    n_pos = np.bincount(np.repeat(np.arange(nE), cnt), weights=rr > 0, minlength=nE)   # numExplicits
    lam = n_pos.astype(np.float64) * reg
    for j in range(k):
        A_[:, j, j] = A_[:, j, j] + lam
    return A_, B


def solve_half(lay, srcF, src_ids, k, reg, alpha):
    """One implicit computeFactors.  Returns (dst float32 [nE][k], the first singular entity or -1)."""
    Am, B = normal_equations(lay, srcF, src_ids, k, reg, alpha)
    y, bad = A.cholesky_solve(Am, B)
    return y.astype(np.float32), int(np.flatnonzero(bad)[0]) if bad.any() else -1


def fit(user, movie, rating, rank=10, max_iter=5, reg_param=0.01, alpha=1.0, seed=0, solver=solve_half,
        init=A.init_user_factors):
    """ALS.fit with implicitPrefs: returns (user ids, user factors, movie ids, movie factors)."""
    uids, mids, by_movie, by_user = A.layouts(user, movie, rating)
    U = init(uids, rank, seed)
    M = np.zeros((len(mids), rank), np.float32)
    for it in range(1, max_iter + 1):
        M, bad = solver(by_movie, U, uids, rank, reg_param, alpha)
        if bad >= 0:
            raise A.SingularError("movie", int(mids[bad]), it)
        U, bad = solver(by_user, M, mids, rank, reg_param, alpha)
        if bad >= 0:
            raise A.SingularError("user", int(uids[bad]), it)
    return uids, U, mids, M


# ---- RankingMetrics ---------------------------------------------------------------------------------------------
def gain(i):
    """1 / ln(i + 2), with the C library's log."""
    return 1.0 / math.log(float(i + 2))


def query_metrics(pred, lab, k):
    """(precision@k, NDCG@k, average precision) of one query, Spark 2.4's loops."""
    pred = [int(x) for x in pred]
    lab_set = set(int(x) for x in lab)
    if not lab_set:
        return 0.0, 0.0, 0.0
    n_prec = min(len(pred), k)
    cnt = 0
    for i in range(n_prec):
        if pred[i] in lab_set:
            cnt += 1
    prec = cnt / k
    n = min(max(len(pred), len(lab_set)), k)
    dcg = max_dcg = 0.0
    for i in range(n):
        g = gain(i)
        if i < len(pred) and pred[i] in lab_set:
            dcg += g
        if i < len(lab_set):
            max_dcg += g
    cnt, prec_sum = 0, 0.0
    for i in range(len(pred)):
        if pred[i] in lab_set:
            cnt += 1
            prec_sum += cnt / (i + 1)
    return prec, dcg / max_dcg, prec_sum / len(lab_set)


def stat_mean(values):
    """StatCounter's mean in order: mu += (x - mu) / n; NaN for no values."""
    mu, n = 0.0, 0
    for x in values:
        n += 1
        mu = mu + (float(x) - mu) / n
    return mu if n else float("nan")


def ranking_metrics(pred_ids, labels, k):
    """(means dict, per-query [n][3]) over queries (pred_ids[q] best first, labels[q] the relevant ids)."""
    per = [query_metrics(p, lab, int(k)) for p, lab in zip(pred_ids, labels)]
    names = ("precision_at_k", "ndcg_at_k", "mean_average_precision")
    return {nm: stat_mean([v[i] for v in per]) for i, nm in enumerate(names)}, np.array(per, np.float64)
