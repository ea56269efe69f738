"""numpy restatement of Spark ML ALS with nonnegative = true: NNLSSolver on the explicit or implicit normal
equations (DESIGN.md section 4.21).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT.  The layouts, init and normal equations are oracle/als.py's and
oracle/als_implicit.py's; only the solve differs.  It restates Spark 2.4's `ALS.NNLSSolver` (fillAtA, then
`NNLS.solve`, then toFloat) and `mllib/optimization/NNLS.scala` from memory; parity with Spark is unpinned.  The
work is vectorised across entities, but every sum of one entity keeps the rule's order (reference BLAS's ddot,
dgemv "N" and daxpy as F2J runs them) with one rounding per operation, and step 7's clip is a scan in i order.
"""
from __future__ import annotations

import numpy as np

from . import als as A
from . import als_implicit as I

WALL = 1 - 1e-14                                            # NNLS.solve's x(i) * (1 - 1e-14)


def iter_max(k):
    return max(400, 20 * k)


def _ddot(a, b):
    """ddot per row: from 0.0, i ascending."""
    s = np.zeros(a.shape[0])
    for i in range(a.shape[1]):
        s = s + a[:, i] * b[:, i]
    return s


def _gemv(Am, v):
    """dgemv "N" per row with beta 0: y = 0, then for each column j with v(j) != 0, y(i) += (1.0 v(j)) A(i,j)."""
    y = np.zeros(v.shape)
    for j in range(v.shape[1]):
        vj = v[:, j]
        y = np.where((vj != 0)[:, None], y + vj[:, None] * Am[:, :, j], y)
    return y


def _stop(step, ndir, nx):
    return np.isnan(step) | (step < 1e-7) | (step > 1e40) | (ndir < 1e-12 * nx) | (ndir < 1e-32)


def nnls(Am, B, mutant=None):
    """NNLS.solve on each system: Am [nE][k][k] the full symmetric matrix (fillAtA's: the packed upper ata mirrored,
    lambda on its diagonal), B [nE][k] atb.  Returns (x double [nE][k], iterations [nE]): the loop ran
    `iterations` times, iter_max(k) when it never stopped.  `mutant` names a deliberate change of the rule (the
    tests use these to show their checks see it): "no_projection", "always_cg", "no_clip", "parallel_clip"."""
    Am = np.asarray(Am, np.float64)
    B = np.asarray(B, np.float64)
    nE, k = B.shape
    x_out = np.zeros((nE, k))
    it_out = np.full(nE, iter_max(k), np.int64)
    live = np.arange(nE)                                    # the entities still iterating, compacted
    A_, b = Am, B
    x = np.zeros((nE, k))
    last_dir = np.zeros((nE, k))
    last_norm = np.zeros(nE)
    last_wall = np.zeros(nE, np.int64)
    with np.errstate(all="ignore"):
        for iterno in range(iter_max(k)):
            if not len(live):
                break
            res = _gemv(A_, x) - b                          # dgemv, then daxpy(-1, atb)
            grad = res.copy()
            if mutant != "no_projection":
                grad[(grad > 0) & (x == 0)] = 0.0
            ngrad = _ddot(grad, grad)
            step = _ddot(grad, res) / (_ddot(_gemv(A_, grad), grad) + 1e-20)
            nx = _ddot(x, x)
            ndir = ngrad.copy()
            d = grad.copy()
            cg = (iterno > last_wall + 1) | (mutant == "always_cg" and iterno > 0)
            if cg.any():
                alpha = ngrad / last_norm
                dcg = np.where((alpha != 0)[:, None], grad + alpha[:, None] * last_dir, grad)   # daxpy skips 0
                dstep = _ddot(dcg, res) / (_ddot(_gemv(A_, dcg), dcg) + 1e-20)
                nd = _ddot(dcg, dcg)
                take = cg & ~_stop(dstep, nd, nx)
                if mutant == "always_cg":
                    take = cg
                d = np.where(take[:, None], dcg, grad)
                step = np.where(take, dstep, step)
                ndir = np.where(take, nd, ngrad)
            done = _stop(step, ndir, nx)
            if mutant == "parallel_clip":                   # each i against the incoming step, the last one wins
                s0 = step
                for i in range(k):
                    step = np.where(s0 * d[:, i] > x[:, i], x[:, i] / d[:, i], step)
            elif mutant != "no_clip":
                for i in range(k):                          # in order: each i sees the step the ones before it left
                    step = np.where(step * d[:, i] > x[:, i], x[:, i] / d[:, i], step)
            sd = step[:, None] * d
            hit = sd > x * WALL
            xn = np.where(hit, 0.0, x - sd)
            last_wall = np.where(hit.any(axis=1), iterno, last_wall)
            # the stopped entities keep their x and leave
            x_out[live[done]] = x[done]
            it_out[live[done]] = iterno
            keep = ~done
            live, A_, b = live[keep], A_[keep], b[keep]
            x, last_dir, last_norm, last_wall = xn[keep], d[keep], ngrad[keep], last_wall[keep]
        x_out[live] = x
    return x_out, it_out


def solve_half(lay, srcF, src_ids, k, reg, alpha=None, mutant=None):
    """One computeFactors with NNLSSolver: the explicit (alpha None) or implicit normal equations, NNLS.solve, then
    toFloat.  Returns (dst float32 [nE][k], -1): there is no singular system."""
    if alpha is None:
        Am, B = A.normal_equations(lay, srcF, k, 0.0 if mutant == "no_lambda" else reg)
    else:
        Am, B = I.normal_equations(lay, srcF, src_ids, k, 0.0 if mutant == "no_lambda" else reg, alpha)
    Am = np.triu(Am) + np.transpose(np.triu(Am, 1), (0, 2, 1))   # fillAtA: mirror the packed upper triangle
    x, _ = nnls(Am, B, None if mutant == "no_lambda" else mutant)
    return x.astype(np.float32), -1


def fit(user, movie, rating, rank=10, max_iter=5, reg_param=0.01, seed=0, implicit_prefs=False, alpha=1.0,
        solver=solve_half, init=A.init_user_factors):
    """ALS.fit with nonnegative = true: returns (user ids, user factors, movie ids, movie factors)."""
    uids, mids, by_movie, by_user = A.layouts(user, movie, rating)
    a = float(alpha) if implicit_prefs else None
    U = init(uids, rank, seed)
    M = np.zeros((len(mids), rank), np.float32)
    for _ in range(max_iter):
        M, _ = solver(by_movie, U, uids, rank, reg_param, a)
        U, _ = solver(by_user, M, mids, rank, reg_param, a)
    return uids, U, mids, M
