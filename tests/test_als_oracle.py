"""ALS's oracles (oracle/als.py, oracle/als_c.c) and the host side of `collab` against known answers.

The fixture is `featureeng_ratings.npz`: 203 150 ratings of users 1..5000 over 952 movies.  DESIGN.md section 4.13
gives the semantics.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest

from oracle import als as A
from oracle import als_cext as X
from oracle.item2vec import splitmix
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import collab

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def fixture_ratings():
    r = np.load(os.path.join(GOLDEN, "featureeng_ratings.npz"))
    return {"userId": r["userId"].astype(np.int32), "movieId": r["movieId"].astype(np.int32),
            "rating": (r["half"] / 2.0).astype(np.float32)}


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def same_fit(a, b):
    for x, y in zip(a, b):
        assert x.shape == y.shape
        assert np.array_equal(bits(x) if x.dtype == np.float32 else x, bits(y) if y.dtype == np.float32 else y)


def hand_cases():
    """name -> (user, movie, rating): the shapes the issue's corner cases need."""
    rng = np.random.default_rng(5)
    cases = {}
    u = rng.integers(1, 40, 600)
    m = rng.integers(1, 30, 600)
    u = np.r_[u, 99]                                       # user 99 has one rating
    m = np.r_[m, 3]
    cases["one_rating_user"] = (u, m, rng.integers(1, 11, len(u)) / 2.0)
    users = np.arange(1, 51)
    cases["movie_rated_by_everyone"] = (np.r_[users, rng.integers(1, 51, 300)], np.r_[np.full(50, 7),
                                        rng.integers(1, 20, 300)], rng.integers(1, 11, 350) / 2.0)
    u = rng.integers(1, 30, 400)
    m = rng.integers(1, 25, 400)
    cases["duplicate_pairs"] = (np.r_[u, u[:60], u[:20]], np.r_[m, m[:60], m[:20]], rng.integers(1, 11, 480) / 2.0)
    cases["sparse_large_ids"] = (rng.choice([5, 70000, 2 ** 31 - 1, 123456789, 42], 300),
                                 rng.choice([0, 2 ** 30, 99999, 17, 2 ** 31 - 2, 31337], 300),
                                 rng.integers(1, 11, 300) / 2.0)
    return cases


# ---- the solve ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("half_step", [0, 1, 3])
def test_each_half_step_solve_matches_linalg_solve(half_step):
    r = fixture_ratings()
    uids, mids, by_movie, by_user = A.layouts(r["userId"], r["movieId"], r["rating"])
    U = X.init_user_factors(uids, 10, 0)
    M = None
    for h in range(half_step + 1):
        lay, src = (by_movie, U) if h % 2 == 0 else (by_user, M)
        Am, B = A.normal_equations(lay, src, 10, 0.01)
        x, bad = A.cholesky_solve(Am, B)
        assert not bad.any()
        if h == half_step:
            full = np.triu(Am) + np.triu(Am, 1).transpose(0, 2, 1)
            ref = np.linalg.solve(full, B[:, :, None])[:, :, 0]
            rel = np.linalg.norm(x - ref, axis=1) / np.linalg.norm(ref, axis=1)
            assert rel.max() < 1e-12, rel.max()
            out, first = X.solve_half(lay, src, 10, 0.01)
            assert first == -1 and np.array_equal(bits(out), bits(x.astype(np.float32)))
        if h % 2 == 0:
            M = x.astype(np.float32)
        else:
            U = x.astype(np.float32)


def test_normal_equations_count_every_rating_with_lambda_n():
    lay = (np.array([0, 3], np.int32), np.array([0, 1, 0], np.int32), np.array([2.0, 0.0, 4.0], np.float32))
    src = np.array([[1.0, 0.0], [0.5, 2.0]], np.float32)
    Am, B = A.normal_equations(lay, src, 2, 0.1)
    lam = 3 * 0.1
    assert np.array_equal(np.triu(Am[0]), [[((1.0 + 0.25) + 1.0) + lam, 0.0 + 1.0], [0, 4.0 + lam]])
    assert np.array_equal(B, [[6.0, 0.0]])                 # rating 0 adds nothing; duplicates count twice


# ---- init -----------------------------------------------------------------------------------------------------
def test_initial_factors_have_unit_norm_and_both_oracles_agree():
    ids = np.array([1, 2, 3, 77, 2 ** 31 - 1, 0], np.int32)
    for rank in (1, 2, 10, 33, 64):
        a = A.init_user_factors(ids, rank, 11)
        assert np.array_equal(bits(a), bits(X.init_user_factors(ids, rank, 11)))
        assert np.abs(np.linalg.norm(a.astype(np.float64), axis=1) - 1).max() < 1e-6
    a = A.init_user_factors(ids, 10, 11)
    assert np.array_equal(a[1], A.init_factor(11, 2, 10))  # keyed by the user id, not its position
    assert not np.array_equal(a, A.init_user_factors(ids, 10, 12))


def test_item_init_is_never_read():
    u, m, r = hand_cases()["one_rating_user"]
    a = A.fit(u, m, r, rank=4, max_iter=2, seed=3)
    junk = np.random.default_rng(0).normal(size=(len(np.unique(m)), 4)).astype(np.float32)
    same_fit(a, A.fit(u, m, r, rank=4, max_iter=2, seed=3, item_init=junk))


# ---- numpy and C oracles --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(hand_cases()))
@pytest.mark.parametrize("rank", [1, 10, 33, 64])
def test_numpy_and_c_oracles_bit_equal_on_hand_built_cases(name, rank):
    u, m, r = hand_cases()[name]
    kw = dict(rank=rank, max_iter=2, reg_param=0.05, seed=rank)
    same_fit(A.fit(u, m, r, **kw), X.fit(u, m, r, **kw))


def test_sparse_ids_and_duplicates_keep_their_rule():
    u, m, r = hand_cases()["duplicate_pairs"]
    uids, mids, by_movie, by_user = A.layouts(u, m, r)
    off, src, rr = by_user
    for e in range(len(uids)):
        s = src[off[e]:off[e + 1]]
        assert np.all(np.diff(s) >= 0)                     # ascending counterpart
        rows = np.flatnonzero(u == uids[e])
        want = rows[np.lexsort((rows, m[rows]))]
        assert np.array_equal(rr[off[e]:off[e + 1]], np.asarray(r, np.float32)[want])   # duplicates in input order
    uids, mids, _, _ = A.layouts(*hand_cases()["sparse_large_ids"])
    assert uids[-1] == 2 ** 31 - 1 and mids[0] == 0 and mids[-1] == 2 ** 31 - 2


@pytest.mark.parametrize("max_iter", [1, 2])
def test_numpy_and_c_oracles_bit_equal_on_the_fixture(max_iter):
    r = fixture_ratings()
    kw = dict(rank=10, max_iter=max_iter, reg_param=0.01, seed=4)
    same_fit(A.fit(r["userId"], r["movieId"], r["rating"], **kw), X.fit(r["userId"], r["movieId"], r["rating"], **kw))


def singular_case():
    """rank 2, reg 0: movie 5 is rated 0 by users 1..3, so its factor is exactly 0; user 9 rated only movie 5, so
    the user's system is all zero and its first pivot is 0."""
    rng = np.random.default_rng(2)
    u = np.r_[1, 2, 3, 9, rng.integers(1, 4, 40)]
    m = np.r_[5, 5, 5, 5, rng.integers(10, 14, 40)]
    r = np.r_[0.0, 0.0, 0.0, 0.0, rng.integers(1, 11, 40) / 2.0]
    return u, m, r


def test_a_singular_system_is_reported_naming_the_entity():
    u, m, r = singular_case()
    for fit in (A.fit, X.fit):
        with pytest.raises(A.SingularError) as e:
            fit(u, m, r, rank=2, max_iter=1, reg_param=0.0, seed=0)
        assert (e.value.side, e.value.entity_id, e.value.iteration) == ("user", 9, 1)
    X.fit(u, m, r, rank=2, max_iter=1, reg_param=0.01, seed=0)   # any lambda > 0 makes it positive definite


# ---- split, drop, recommend -----------------------------------------------------------------------------------
def test_random_split_follows_the_rule():
    n, seed = 5000, 7
    parts = collab.random_split(n, (0.8, 0.2), seed)
    u = np.array([(splitmix(seed, i) >> 11) * 2.0 ** -53 for i in range(n)])
    assert np.array_equal(parts[0], np.flatnonzero(u < 0.8)) and np.array_equal(parts[1], np.flatnonzero(u >= 0.8))
    assert abs(len(parts[0]) / n - 0.8) < 0.03
    p3 = collab.random_split(n, (1, 1, 2), seed)
    assert np.array_equal(p3[0], np.flatnonzero(u < 0.25))
    assert np.array_equal(p3[1], np.flatnonzero((u >= 0.25) & (u < 0.5)))
    assert sum(len(p) for p in p3) == n
    with pytest.raises(ValueError):
        collab.random_split(n, (0.5, -0.5))


def test_transform_drops_cold_rows_and_predicts_the_float_dot():
    rng = np.random.default_rng(1)
    uf = rng.normal(size=(3, 5)).astype(np.float32)
    mf = rng.normal(size=(4, 5)).astype(np.float32)
    model = collab.AlsModel(np.array([2, 5, 9], np.int32), uf, np.array([1, 3, 4, 8], np.int32), mf)
    test = {"userId": np.array([5, 6, 2, 9, 9, 1]), "movieId": np.array([3, 3, 8, 2, 1, 1])}
    rows, pred = model.transform(test)
    assert rows.tolist() == [0, 2, 4]
    want = A.predict(uf[[1, 0, 2]], mf[[1, 3, 0]])
    assert np.array_equal(bits(pred), bits(want))
    s = np.float32(0)
    for d in range(5):
        s = np.float32(s + np.float32(uf[1, d] * mf[1, d]))
    assert bits(pred[:1])[0] == bits(np.array([s]))[0]


def test_rmse_is_regression_metrics():
    lab = np.array([4.0, 3.5, 1.0], np.float32)
    pred = np.array([3.9, 3.0, 2.5], np.float32)
    d = lab.astype(np.float64) - pred.astype(np.float64)
    ss = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
    assert collab.rmse(lab, pred) == math.sqrt(math.sqrt(ss) ** 2 / 3) == A.rmse(lab, pred)


def test_recommend_ties_go_to_the_lower_destination_id():
    rng = np.random.default_rng(3)
    dst = rng.normal(size=(40, 6)).astype(np.float32)
    dst[[5, 17, 30]] = dst[11]                             # four destinations with the same score for everyone
    ids = np.arange(100, 140, dtype=np.int32)
    src = rng.normal(size=(9, 6)).astype(np.float32)
    src[3] = 0                                             # every score 0: the lowest ids win
    for num in (1, 4, 10, 40, 128):
        a = A.recommend(src, ids, dst, num)
        b = X.recommend(src, ids, dst, num)
        assert np.array_equal(a[0], b[0]) and np.array_equal(bits(a[1]), bits(b[1]))
    ids_, sc = X.recommend(src, ids, dst, 40)
    assert ids_[3, :10].tolist() == list(range(100, 110))
    for row in range(9):
        where = {int(x): i for i, x in enumerate(ids_[row])}
        assert where[105] < where[111] < where[117] < where[130]
        if row != 3:                                       # adjacent, unless every score ties
            assert where[130] - where[105] == 3
        assert all(np.diff(sc[row].astype(np.float64)) <= 0)


# ---- the ABI's device-free rejections ---------------------------------------------------------------------------
def _raw_fit(u, m, r, rank=10, max_iter=5, reg=0.01, cap=8):
    lib = _lib.load()
    u, m = np.ascontiguousarray(u, np.int32), np.ascontiguousarray(m, np.int32)
    r = np.ascontiguousarray(r, np.float32)
    p = _lib.SrsAlsParams(rank, max_iter, reg, 0)
    room = max(cap, 1)
    ui, mi = np.zeros(room, np.int32), np.zeros(room, np.int32)
    uf, mf = np.zeros((room, 64), np.float32), np.zeros((room, 64), np.float32)
    nu, nm = C.c_int32(-1), C.c_int32(-1)
    rc = lib.srs_als_fit_host(u.ctypes.data, m.ctypes.data, r.ctypes.data, len(u), C.byref(p), 0, cap, cap,
                              ui.ctypes.data, uf.ctypes.data, C.byref(nu), mi.ctypes.data, mf.ctypes.data,
                              C.byref(nm))
    return rc, nu.value, nm.value


def _raw_recommend(src, ids, dst, rank, num):
    lib = _lib.load()
    src, dst = np.ascontiguousarray(src, np.float32), np.ascontiguousarray(dst, np.float32)
    ids = np.ascontiguousarray(ids, np.int32)
    oi = np.zeros(max(1, len(src) * num), np.int32)
    os_ = np.zeros(max(1, len(src) * num), np.float32)
    return lib.srs_als_recommend_host(src.ctypes.data, len(src), ids.ctypes.data, dst.ctypes.data, len(ids), rank,
                                      num, 0, oi.ctypes.data, os_.ctypes.data)


def test_fit_rejects_bad_inputs_before_any_device_call():
    u, m, r = [1, 2], [3, 4], [4.0, 5.0]
    INV = _lib.SRS_ERR_INVALID
    assert _raw_fit(u, m, r, rank=0) == (INV, 0, 0)
    assert _raw_fit(u, m, r, rank=65)[0] == INV
    assert _raw_fit(u, m, r, max_iter=0)[0] == INV
    assert _raw_fit(u, m, r, reg=-0.1)[0] == INV
    assert _raw_fit(u, m, r, reg=float("nan"))[0] == INV
    assert _raw_fit(u, m, r, reg=float("inf"))[0] == INV
    assert _raw_fit([1, -2], m, r)[0] == INV
    assert _raw_fit(u, [3, -1], r)[0] == INV
    assert _raw_fit(u, m, [4.0, float("nan")])[0] == INV
    assert _raw_fit([], [], [])[0] == INV
    assert _raw_fit(u, m, r, cap=-1)[0] == INV
    lib = _lib.load()
    p = _lib.SrsAlsParams(10, 5, 0.01, 0)
    nu, nm = C.c_int32(0), C.c_int32(0)
    assert lib.srs_als_fit_host(None, None, None, 2, C.byref(p), 0, 0, 0, None, None, C.byref(nu), None, None,
                                C.byref(nm)) == INV
    assert lib.srs_als_fit_host(None, None, None, 21000001, C.byref(p), 0, 0, 0, None, None, C.byref(nu), None,
                                None, C.byref(nm)) == INV
    assert "rank" in lib.srs_last_error().decode() or "n_ratings" in lib.srs_last_error().decode()


def test_recommend_rejects_bad_inputs_before_any_device_call():
    INV = _lib.SRS_ERR_INVALID
    s, d = np.ones((2, 3)), np.ones((4, 3))
    assert _raw_recommend(s, [1, 2, 3, 4], d, 3, 0) == INV
    assert _raw_recommend(s, [1, 2, 3, 4], d, 3, 129) == INV
    assert _raw_recommend(s, [1, 2, 3, 4], d, 0, 5) == INV
    assert _raw_recommend(s, [1, 2, 3, 4], d, 65, 5) == INV
    assert _raw_recommend(s, [1, 3, 3, 4], d, 3, 5) == INV            # ids not strictly ascending
    bad = d.copy()
    bad[2, 1] = np.inf
    assert _raw_recommend(s, [1, 2, 3, 4], bad, 3, 5) == INV
    assert _raw_recommend(np.full((2, 3), np.nan), [1, 2, 3, 4], d, 3, 5) == INV
