"""Implicit-feedback ALS and RankingMetrics: the oracles (oracle/als_implicit.py, oracle/als_implicit_c.c) against
known answers, and the ABI's device-free rejections.  DESIGN.md section 4.17 gives the semantics."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import als as A
from oracle import als_cext as X
from oracle import als_implicit as I
from oracle import als_implicit_cext as XI
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import collab

from test_als_oracle import bits, fixture_ratings, same_fit


def implicit_cases():
    """name -> (user, movie, rating): the corner cases of the implicit normal equations."""
    rng = np.random.default_rng(11)
    cases = {}
    # more users and movies than rank 64, so that YtY alone (alpha 0, no positive rating) stays positive definite
    u = rng.integers(0, 150, 3000)                         # users 0..149: every YtY block
    m = rng.choice([i for i in range(1, 300) if i % 10 != 7], 3000)   # no movie in block 7
    r = rng.integers(1, 11, 3000) / 2.0
    r[:150] = 0.0                                          # zero ratings: no effect
    r[150:300] = -rng.integers(1, 6, 150) / 2.0            # negative ratings: confidence only
    u = np.r_[u, u[400:440], 977, 977, 977]                # duplicate pairs; user 977 rates only <= 0
    m = np.r_[m, m[400:440], 3, 5, 3]
    r = np.r_[r, r[400:440], 0.0, -2.0, -0.5]
    cases["corners"] = (u, m, r)
    cases["sparse_large_ids"] = (rng.choice([5, 70000, 2 ** 31 - 1, 123456789, 42, 8, 19, 2 ** 30 + 3], 400),
                                 rng.choice([0, 2 ** 30, 99999, 17, 2 ** 31 - 2, 31337, 64, 6], 400),
                                 rng.integers(1, 11, 400) / 2.0)
    return cases


def _dense_system(lay, srcF, k, reg, alpha):
    """The issue's formula in plain numpy, in any order: (YtY + sum c1 y y^T + lambda n+ I, sum_{r>0} (1 + c1) y)."""
    off, src, r = lay
    Y = srcF.astype(np.float64)
    yty = Y.T @ Y
    out_a, out_b = [], []
    for e in range(len(off) - 1):
        a, b, npos = yty.copy(), np.zeros(k), 0
        for p in range(off[e], off[e + 1]):
            y, rv = Y[src[p]], float(r[p])
            c1 = alpha * abs(rv)
            a += c1 * np.outer(y, y)
            if rv > 0:
                b += (1 + c1) * y
                npos += 1
        out_a.append(a + reg * npos * np.eye(k))
        out_b.append(b)
    return np.array(out_a), np.array(out_b)


def _check_half_steps(u, m, r, k, reg, alpha, half_steps, seed=0):
    uids, mids, by_movie, by_user = A.layouts(u, m, r)
    U = X.init_user_factors(uids, k, seed)
    M = None
    for h in range(half_steps):
        lay, src, ids = (by_movie, U, uids) if h % 2 == 0 else (by_user, M, mids)
        Am, B = I.normal_equations(lay, src, ids, k, reg, alpha)
        x, bad = A.cholesky_solve(Am, B)
        assert not bad.any()
        Ad, Bd = _dense_system(lay, src, k, reg, alpha)
        ref = np.linalg.solve(Ad, Bd[:, :, None])[:, :, 0]
        nz = np.linalg.norm(ref, axis=1) > 0
        rel = np.linalg.norm(x - ref, axis=1)[nz] / np.linalg.norm(ref, axis=1)[nz]
        assert rel.max() < 1e-12, (h, rel.max())
        assert np.array_equal(x[~nz], ref[~nz])            # no positive rating: an exactly zero solution
        out, first = XI.solve_half(lay, src, ids, k, reg, alpha)
        assert first == -1 and np.array_equal(bits(out), bits(x.astype(np.float32)))
        if h % 2 == 0:
            M = x.astype(np.float32)
        else:
            U = x.astype(np.float32)


# ---- the solve ------------------------------------------------------------------------------------------------
def test_each_half_step_on_the_fixture_matches_linalg_solve():
    r = fixture_ratings()
    _check_half_steps(r["userId"], r["movieId"], r["rating"], 10, 0.01, 1.0, 2)


@pytest.mark.parametrize("name", sorted(implicit_cases()))
@pytest.mark.parametrize("alpha", [0.0, 1.0, 40.0])
def test_each_half_step_on_hand_built_cases_matches_linalg_solve(name, alpha):
    u, m, r = implicit_cases()[name]
    _check_half_steps(u, m, r, 4, 0.05, alpha, 4, seed=3)


def test_the_hand_built_case_reaches_its_corners():
    u, m, r = implicit_cases()["corners"]
    assert {int(x) % 10 for x in np.unique(u)} == set(range(10))
    assert 7 not in {int(x) % 10 for x in np.unique(m)}
    assert np.any(r == 0) and np.any(r < 0)
    pairs = list(zip(u.tolist(), m.tolist()))
    assert len(set(pairs)) < len(pairs)
    assert np.all(r[u == 977] <= 0)


def test_one_entity_by_hand_zero_negative_and_duplicate_ratings():
    """Movie 0 rated 2.0, -1.0, 0.0 and 2.0 again (a duplicate pair) by sources 0, 1, 0, 0; alpha 0.5, reg 0.1."""
    src = np.array([[1.0, 0.0], [0.5, 2.0]], np.float32)
    ids = np.array([3, 14], np.int32)                      # blocks 3 and 4
    lay = (np.array([0, 4], np.int32), np.array([0, 1, 0, 0], np.int32),
           np.array([2.0, -1.0, 0.0, 2.0], np.float32))
    Am, B = I.normal_equations(lay, src, ids, 2, 0.1, 0.5)
    yty = np.array([[1.0 + 0.25, 1.0], [1.0, 4.0]])        # ((0 + B3) + B4): y0 y0^T + y1 y1^T
    a = yty.copy()
    a = a + 1.0 * np.array([[1.0, 0.0], [0.0, 0.0]])       # r 2.0: c1 = 1.0 (x(1) = 0 skips column 1)
    a = a + np.array([[0.5 * 0.25, 0.5 * 1.0], [0, 0.5 * 4.0]])   # r -1.0: c1 = 0.5, no preference, not counted
    a = a + 1.0 * np.array([[1.0, 0.0], [0.0, 0.0]])       # r 0.0 adds nothing; the duplicate 2.0 adds again
    lam = 2 * 0.1                                          # two positive ratings
    want = np.triu(a) + lam * np.eye(2)
    assert np.array_equal(np.triu(Am[0]), want)
    assert np.array_equal(B, [[2.0 * 1.0 + 2.0 * 1.0, 0.0]])   # (1 + c1) y for each positive rating


def test_a_zero_rating_changes_no_bit():
    u, m, r = implicit_cases()["corners"]
    keep = r != 0
    for fit in (I.fit, XI.fit):
        a = fit(u, m, r, rank=5, max_iter=2, reg_param=0.05, alpha=2.0, seed=1)
        b = fit(u[keep], m[keep], r[keep], rank=5, max_iter=2, reg_param=0.05, alpha=2.0, seed=1)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])   # every id keeps another rating
        same_fit(a, b)


def test_all_non_positive_ratings_get_lambda_zero_and_a_zero_factor():
    u, m, r = implicit_cases()["corners"]
    uids, U, mids, M = XI.fit(u, m, r, rank=4, max_iter=1, reg_param=0.05, alpha=1.0)
    assert np.all(U[np.searchsorted(uids, 977)] == 0)       # atb = 0: dpptrs of a zero right-hand side


# ---- YtY ------------------------------------------------------------------------------------------------------
def _yty_by_hand(ids, Y, order):
    k = Y.shape[1]
    part = [[[0.0] * k for _ in range(k)] for _ in range(10)]
    for e in sorted(range(len(ids)), key=lambda e: ids[e]):
        b, y = int(ids[e]) % 10, [float(v) for v in Y[e]]
        for j in range(k):
            if y[j] == 0.0:
                continue
            for i in range(j + 1):
                part[b][i][j] = part[b][i][j] + y[i] * (1.0 * y[j])
    out = [[0.0] * k for _ in range(k)]
    for b in order:
        for j in range(k):
            for i in range(j + 1):
                out[i][j] = out[i][j] + 1.0 * part[b][i][j]
    return np.array([out[i][j] for j in range(k) for i in range(j + 1)])


def _packed(full):
    k = full.shape[0]
    return np.array([full[i, j] for j in range(k) for i in range(j + 1)])


def test_yty_follows_the_block_rule_bit_for_bit():
    rng = np.random.default_rng(6)
    ids = np.sort(rng.choice(10 ** 6, 700, replace=False)).astype(np.int32)
    ids = ids[ids % 10 != 4]                               # one block with no entity
    Y = rng.normal(size=(len(ids), 7)).astype(np.float32)
    Y[::13, 2] = 0.0                                       # dspr skips the zero columns
    want = _yty_by_hand(ids, Y, range(10))
    assert np.array_equal(_packed(I.yty(ids, Y)), want)
    assert np.array_equal(XI.yty(ids, Y), want)


def test_the_merge_order_is_visible_in_the_bits():
    rng = np.random.default_rng(6)
    ids = np.arange(1, 2001, dtype=np.int32)
    Y = rng.normal(size=(len(ids), 10)).astype(np.float32)
    rev = tuple(range(9, -1, -1))
    assert np.array_equal(XI.yty(ids, Y, rev), _yty_by_hand(ids, Y, rev))
    assert not np.array_equal(XI.yty(ids, Y), XI.yty(ids, Y, rev))
    assert np.array_equal(_packed(I.yty(ids, Y, rev)), XI.yty(ids, Y, rev))
    assert np.allclose(XI.yty(ids, Y), XI.yty(ids, Y, rev), rtol=1e-13, atol=1e-12)


# ---- numpy and C oracles --------------------------------------------------------------------------------------
@pytest.mark.parametrize("rank", [1, 10, 33, 64])
@pytest.mark.parametrize("max_iter", [1, 2])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 40.0])
def test_numpy_and_c_oracles_bit_equal(rank, max_iter, alpha):
    for u, m, r in implicit_cases().values():
        kw = dict(rank=rank, max_iter=max_iter, reg_param=0.05, alpha=alpha, seed=rank)
        same_fit(I.fit(u, m, r, **kw), XI.fit(u, m, r, **kw))


@pytest.mark.parametrize("max_iter", [1, 2])
def test_numpy_and_c_oracles_bit_equal_on_the_fixture(max_iter):
    r = fixture_ratings()
    kw = dict(rank=10, max_iter=max_iter, reg_param=0.01, alpha=1.0, seed=4)
    same_fit(I.fit(r["userId"], r["movieId"], r["rating"], **kw),
             XI.fit(r["userId"], r["movieId"], r["rating"], **kw))


def implicit_singular_case():
    """rank 2, one user (id 9): YtY = y y^T has rank 1, and its second pivot is exactly 0 (y0 y1 / |y0| = +-y1 and
    y1^2 are exact in double).  Movie 5 is rated 0 - no term, lambda 0 - so its system is YtY alone; movie 6, rated
    4.0, is regular."""
    return np.array([9, 9]), np.array([6, 5]), np.array([4.0, 0.0])


def test_a_singular_implicit_system_is_reported_naming_the_entity():
    u, m, r = implicit_singular_case()
    for fit in (I.fit, XI.fit):
        with pytest.raises(A.SingularError) as e:
            fit(u, m, r, rank=2, max_iter=1, reg_param=0.01, alpha=1.0, seed=0)
        assert (e.value.side, e.value.entity_id, e.value.iteration) == ("movie", 5, 1)


# ---- RankingMetrics -------------------------------------------------------------------------------------------
def _g(i):
    return 1.0 / math.log(i + 2.0)


def _both(pred, labels, k):
    """The numpy oracle's (means, per-query [n][3]), checked equal to the C oracle's."""
    means, per = I.ranking_metrics(pred, labels, k)
    off = np.r_[0, np.cumsum([len(x) for x in labels])].astype(np.int32)
    ids = np.concatenate([np.asarray(x, np.int64) for x in labels]).astype(np.int32) if labels else []
    cm, cper = XI.ranking_metrics(np.asarray(pred, np.int32).reshape(len(labels), -1), off, ids, k)
    got = [means["precision_at_k"], means["ndcg_at_k"], means["mean_average_precision"]]
    assert np.array_equal(np.array(got), cm, equal_nan=True)
    assert np.array_equal(per.T if len(per) else per.reshape(3, 0), cper)
    return means, per


def test_an_empty_label_set_scores_zero_and_counts():
    means, per = _both([[1, 2, 3], [4, 5, 6]], [[], [4]], 3)
    assert per[0].tolist() == [0.0, 0.0, 0.0]
    assert per[1].tolist() == [1 / 3, 1.0, 1.0]
    assert means["precision_at_k"] == 0.0 + (1 / 3 - 0.0) / 2


def test_fewer_predictions_than_k():
    pred, lab, k = [7, 1, 9], [9, 2, 7], 5                 # L = 3 < k, hits at 0 and 2
    _, per = _both([pred], [lab], k)
    assert per[0, 0] == 2 / 5                              # over k, not L
    dcg = _g(0) + _g(2)
    max_dcg = (_g(0) + _g(1)) + _g(2)                      # min(max(3, 3), 5) = 3 positions
    assert per[0, 1] == dcg / max_dcg
    assert per[0, 2] == (1 / 1 + 2 / 3) / 3


def test_more_predictions_than_k_and_map_over_the_whole_list():
    pred, lab, k = [5, 6, 1, 2, 3, 4], [1, 4], 2           # hits at 2 and 5, both past k
    _, per = _both([pred], [lab], k)
    assert per[0, 0] == 0.0 and per[0, 1] == 0.0
    assert per[0, 2] == (1 / 3 + 2 / 6) / 2                # MAP reads every prediction


def test_more_labels_than_k():
    pred, lab, k = [1, 2], [1, 2, 3, 4, 5, 6], 4           # |lab| = 6 > k: maxDcg over k positions
    _, per = _both([pred], [lab], k)
    assert per[0, 0] == 2 / 4
    assert per[0, 1] == (_g(0) + _g(1)) / (((_g(0) + _g(1)) + _g(2)) + _g(3))
    assert per[0, 2] == (1 / 1 + 2 / 2) / 6


def test_duplicate_labels_collapse():
    a = _both([[3, 8, 4]], [[4, 4, 3, 3, 3]], 3)[1]
    b = _both([[3, 8, 4]], [[3, 4]], 3)[1]
    assert np.array_equal(a, b)
    assert a[0, 2] == (1 / 1 + 2 / 3) / 2


def test_a_query_with_all_hits():
    _, per = _both([[4, 2, 9]], [[9, 4, 2]], 3)
    assert per[0].tolist() == [1.0, 1.0, 1.0]


def test_the_mean_is_statcounters():
    hits = [5, 0, 3, 5, 4, 4, 0]                           # per-query precisions h / 10 at k = 10
    vals = [h / 10 for h in hits]
    mu = 0.0
    for n, x in enumerate(vals, 1):
        mu = mu + (x - mu) / n
    assert mu == 0.30000000000000004 and sum(vals) / len(vals) == 0.3   # the naive mean differs
    pred = [list(range(10)) for _ in hits]
    labels = [list(range(h)) + [99] * (h == 0) for h in hits]   # a miss keeps the zero-hit label sets non-empty
    means, per = _both(pred, labels, 10)
    assert per[:, 0].tolist() == vals and means["precision_at_k"] == mu


def test_no_query_gives_nan():
    means, _ = I.ranking_metrics([], [], 10)
    assert all(math.isnan(v) for v in means.values())


# ---- the ABI's device-free rejections ---------------------------------------------------------------------------
def _raw_implicit(u, m, r, rank=10, max_iter=5, reg=0.01, alpha=1.0, cap=8):
    lib = _lib.load()
    u, m = np.ascontiguousarray(u, np.int32), np.ascontiguousarray(m, np.int32)
    r = np.ascontiguousarray(r, np.float32)
    p = _lib.SrsAlsParams(rank, max_iter, reg, 0)
    ui, mi = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    uf, mf = np.zeros((cap, 64), np.float32), np.zeros((cap, 64), np.float32)
    nu, nm = C.c_int32(-1), C.c_int32(-1)
    rc = lib.srs_als_fit_implicit_host(u.ctypes.data, m.ctypes.data, r.ctypes.data, len(u), C.byref(p), 0, cap, cap,
                                       ui.ctypes.data, uf.ctypes.data, C.byref(nu), mi.ctypes.data, mf.ctypes.data,
                                       C.byref(nm), alpha)
    return rc, nu.value, nm.value, lib.srs_last_error().decode()


def test_implicit_fit_rejects_bad_inputs_before_any_device_call():
    u, m, r = [1, 2], [3, 4], [4.0, 5.0]
    INV = _lib.SRS_ERR_INVALID
    for kw, word in ((dict(alpha=-0.5), "alpha"), (dict(alpha=float("nan")), "alpha"),
                     (dict(alpha=float("inf")), "alpha"), (dict(rank=0), "rank"), (dict(rank=65), "rank"),
                     (dict(max_iter=0), "max_iter"), (dict(reg=-1.0), "reg_param")):
        rc, nu, nm, msg = _raw_implicit(u, m, r, **kw)
        assert (rc, nu, nm) == (INV, 0, 0) and word in msg, (kw, msg)
    for bad in (float("nan"), float("inf"), -float("inf")):
        rc, _, _, msg = _raw_implicit(u, m, [4.0, bad])
        assert rc == INV and "not finite" in msg
    assert _raw_implicit([1, -2], m, r)[0] == INV
    assert _raw_implicit([], [], [])[0] == INV


def _raw_ranking(pred, off, ids, k):
    lib = _lib.load()
    pred = np.ascontiguousarray(pred, np.int32)
    off = np.ascontiguousarray(off, np.int32)
    ids = np.ascontiguousarray(ids if len(ids) else [0], np.int32)
    means = np.zeros(3)
    n = len(off) - 1
    return lib.srs_ranking_metrics_host(pred.ctypes.data, n, pred.shape[1] if pred.ndim == 2 else 0,
                                        off.ctypes.data, ids.ctypes.data, k, 0, None, means.ctypes.data), means


def test_ranking_metrics_reject_bad_inputs_before_any_device_call():
    INV = _lib.SRS_ERR_INVALID
    assert _raw_ranking([[1, 2]], [0, 1], [1], 0)[0] == INV
    assert _raw_ranking([[1, 2]], [1, 1], [1], 3)[0] == INV               # offsets must start at 0
    assert _raw_ranking([[1, 2], [3, 4]], [0, 2, 1], [1, 2], 3)[0] == INV  # and never decrease
    rc, means = _raw_ranking(np.zeros((0, 3)), [0], [], 3)                 # no query: NaN, no device needed
    assert rc == _lib.SRS_OK and np.all(np.isnan(means))
    with pytest.raises(ValueError):
        collab.ranking_metrics([[1, 2]], [[1], [2]], 3)
    with pytest.raises(ValueError):
        collab.ranking_metrics([[1, 2]], (np.array([0, 3]), np.array([1, 2])), 3)
