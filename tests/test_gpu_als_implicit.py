"""Implicit-feedback ALS and RankingMetrics on the device (`collab`, csrc/als.cu) against the C oracles, bit for
bit."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import als_cext as X
from oracle import als_implicit_cext as XI
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import collab
from sparrowrecsys_b200.model import launch_count

from test_als_implicit_oracle import _raw_implicit, implicit_cases, implicit_singular_case
from test_als_oracle import GOLDEN, fixture_ratings, same_fit

pytestmark = pytest.mark.gpu


def _dev(r, **kw):
    m = collab.als(r, implicit_prefs=True, **kw)
    return m.user_ids, m.user_factors, m.item_ids, m.item_factors


def _check(u, m, r, **kw):
    dev = _dev({"userId": u, "movieId": m, "rating": r}, **kw)
    same_fit(dev, XI.fit(u, m, np.asarray(r, np.float32), **kw))
    return dev


@pytest.fixture(scope="module")
def fixture():
    return fixture_ratings()


@pytest.mark.parametrize("seed", [0, 1])
def test_the_scripts_implicit_fit_is_bit_equal_to_the_c_oracle(fixture, seed):
    tr, _ = collab.random_split(len(fixture["userId"]), (0.8, 0.2), seed)
    sub = {k: v[tr] for k, v in fixture.items()}
    _check(sub["userId"], sub["movieId"], sub["rating"], rank=10, max_iter=5, reg_param=0.01, alpha=1.0, seed=seed)


@pytest.mark.parametrize("rank", [1, 16, 32, 33, 64])
@pytest.mark.parametrize("max_iter", [1, 2])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 40.0])
def test_ranks_iterations_and_alphas_bit_equal_to_the_c_oracle(fixture, rank, max_iter, alpha):
    _check(fixture["userId"], fixture["movieId"], fixture["rating"], rank=rank, max_iter=max_iter, reg_param=0.01,
           alpha=alpha, seed=rank)


@pytest.mark.parametrize("name", sorted(implicit_cases()))
@pytest.mark.parametrize("rank", [1, 10, 33, 64])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 40.0])
def test_hand_built_cases_bit_equal_to_the_c_oracle(name, rank, alpha):
    u, m, r = implicit_cases()[name]
    _check(u, m, r, rank=rank, max_iter=2, reg_param=0.05, alpha=alpha, seed=rank)


def test_repeat_runs_give_the_same_bits(fixture):
    a = _dev(fixture, rank=12, max_iter=2, alpha=3.0, seed=5)
    same_fit(a, _dev(fixture, rank=12, max_iter=2, alpha=3.0, seed=5))


def test_one_yty_merge_and_solve_per_half_step():
    u, m, r = implicit_cases()["corners"]
    n0 = launch_count()
    collab.als({"userId": u, "movieId": m, "rating": r}, rank=8, max_iter=3, implicit_prefs=True)
    n1 = launch_count()
    collab.als({"userId": u, "movieId": m, "rating": r}, rank=8, max_iter=1, implicit_prefs=True)
    assert (n1 - n0) - (launch_count() - n1) == 2 * 2 * 3       # two more iterations: 2 half-steps x 3 launches


def test_a_singular_implicit_system_names_the_entity_and_writes_nothing():
    u, m, r = implicit_singular_case()
    lib = _lib.load()
    u32, m32, r32 = (np.ascontiguousarray(x, t) for x, t in ((u, np.int32), (m, np.int32), (r, np.float32)))
    p = _lib.SrsAlsParams(2, 1, 0.01, 0)
    ui, mi = np.full(8, -7, np.int32), np.full(8, -7, np.int32)
    uf, mf = np.full((8, 2), 3.5, np.float32), np.full((8, 2), 3.5, np.float32)
    nu, nm = C.c_int32(-1), C.c_int32(-1)
    rc = lib.srs_als_fit_implicit_host(u32.ctypes.data, m32.ctypes.data, r32.ctypes.data, len(u32), C.byref(p), 0,
                                       8, 8, ui.ctypes.data, uf.ctypes.data, C.byref(nu), mi.ctypes.data,
                                       mf.ctypes.data, C.byref(nm), 1.0)
    assert rc == _lib.SRS_ERR_INVALID
    msg = lib.srs_last_error().decode()
    assert "movie 5" in msg and "iteration 1" in msg, msg
    assert nu.value == 0 and nm.value == 0
    assert np.all(ui == -7) and np.all(mi == -7) and np.all(uf == 3.5) and np.all(mf == 3.5)
    with pytest.raises(ValueError, match="movie 5"):
        collab.als({"userId": u, "movieId": m, "rating": r}, rank=2, max_iter=1, implicit_prefs=True)


def test_the_default_call_is_the_explicit_fit(fixture):
    lib = _lib.load()
    u, m, r = (np.ascontiguousarray(fixture[c], t) for c, t in (("userId", np.int32), ("movieId", np.int32),
                                                                ("rating", np.float32)))
    cu, cm = len(np.unique(u)), len(np.unique(m))
    p = _lib.SrsAlsParams(10, 2, 0.01, 3)
    ui, mi = np.zeros(cu, np.int32), np.zeros(cm, np.int32)
    uf, mf = np.zeros((cu, 10), np.float32), np.zeros((cm, 10), np.float32)
    nu, nm = C.c_int32(0), C.c_int32(0)
    assert lib.srs_als_fit_host(u.ctypes.data, m.ctypes.data, r.ctypes.data, len(u), C.byref(p), 0, cu, cm,
                                ui.ctypes.data, uf.ctypes.data, C.byref(nu), mi.ctypes.data, mf.ctypes.data,
                                C.byref(nm)) == _lib.SRS_OK
    for kw in ({}, {"implicit_prefs": False}, {"implicit_prefs": False, "alpha": 7.0}):
        d = collab.als(fixture, rank=10, max_iter=2, reg_param=0.01, seed=3, **kw)
        same_fit((d.user_ids, d.user_factors, d.item_ids, d.item_factors), (ui, uf, mi, mf))


def test_rejections_launch_nothing():
    n0 = launch_count()
    assert _raw_implicit([1, 2], [3, 4], [4.0, 5.0], alpha=-1.0)[0] == _lib.SRS_ERR_INVALID
    assert _raw_implicit([1, 2], [3, 4], [4.0, float("nan")])[0] == _lib.SRS_ERR_INVALID
    with pytest.raises(ValueError):
        collab.ranking_metrics([[1, 2]], [[1]], 0)
    assert launch_count() == n0


# ---- RankingMetrics ---------------------------------------------------------------------------------------------
def _csr(labels):
    off = np.r_[0, np.cumsum([len(x) for x in labels])].astype(np.int32)
    ids = np.concatenate([np.asarray(x, np.int64) for x in labels]).astype(np.int32)
    return off, ids


def _same_metrics(got, means):
    assert [got["precision_at_k"], got["ndcg_at_k"], got["mean_average_precision"]] == means.tolist()


@pytest.fixture(scope="module")
def implicit_model(fixture):
    tr, te = collab.random_split(len(fixture["userId"]), (0.8, 0.2), 0)
    sub = {k: v[tr] for k, v in fixture.items()}
    test = {k: v[te] for k, v in fixture.items()}
    return collab.als(sub, implicit_prefs=True), test


@pytest.mark.parametrize("k", [1, 10, 128])
def test_model_ranking_metrics_equal_the_oracles(implicit_model, k):
    model, test = implicit_model
    for threshold in (0.0, 3.5):
        users, rows, (off, ids) = model.ranking_queries(test, threshold)
        pred, _ = X.recommend(model.user_factors[rows], model.item_ids, model.item_factors, k)
        means, _ = XI.ranking_metrics(pred, off, ids, k)
        _same_metrics(model.ranking_metrics(test, k, threshold), means)


def test_k_beyond_the_movie_count():
    u, m, r = implicit_cases()["sparse_large_ids"]              # 8 movies
    model = collab.als({"userId": u, "movieId": m, "rating": r}, rank=4, max_iter=2, implicit_prefs=True)
    test = {"userId": u[::3], "movieId": m[::3], "rating": r[::3]}
    for k in (7, 8, 9, 100):
        users, rows, (off, ids) = model.ranking_queries(test)
        pred, _ = X.recommend(model.user_factors[rows], model.item_ids, model.item_factors, k)
        assert pred.shape[1] == min(k, 8)
        _same_metrics(model.ranking_metrics(test, k), XI.ranking_metrics(pred, off, ids, k)[0])


@pytest.mark.parametrize("k", [1, 10, 128, 1000])
def test_ranking_metrics_on_random_lists_equal_the_oracle(k):
    rng = np.random.default_rng(k)
    n, L = 3000, 150
    pred = np.stack([rng.choice(400, L, replace=False) for _ in range(n)]).astype(np.int32)
    sizes = rng.integers(0, 300, n)
    sizes[::17] = 0                                            # empty label sets
    labels = [rng.integers(0, 400, s) for s in sizes]         # duplicates included
    labels[5] = pred[5]                                        # every prediction a hit
    means, _ = XI.ranking_metrics(pred, *_csr(labels), k)
    _same_metrics(collab.ranking_metrics(pred, labels, k), means)
    _same_metrics(collab.ranking_metrics(pred, _csr(labels), k), means)


def test_ranking_metrics_repeat_and_edges():
    pred = np.array([[3, 1, 2], [5, 6, 7]], np.int32)
    a = collab.ranking_metrics(pred, [[1, 1, 9], []], 2)
    assert a == collab.ranking_metrics(pred, [[1, 1, 9], []], 2)
    _same_metrics(a, XI.ranking_metrics(pred, *_csr([[1, 1, 9], []]), 2)[0])
    empty = np.zeros((2, 0), np.int32)                          # L = 0
    _same_metrics(collab.ranking_metrics(empty, [[1], [2, 3]], 4),
                  XI.ranking_metrics(empty, *_csr([[1], [2, 3]]), 4)[0])


# ---- the script's --implicit sequence ---------------------------------------------------------------------------
def test_the_implicit_command_gives_the_recorded_output(tmp_path, capsys, fixture):
    with open(os.path.join(GOLDEN, "als_implicit.json")) as f:
        g = json.load(f)
    path = tmp_path / "ratings.csv"
    with open(path, "w") as f:
        f.write("userId,movieId,rating,timestamp\n")
        for row in zip(fixture["userId"].tolist(), fixture["movieId"].tolist(), fixture["rating"].tolist()):
            f.write("%d,%d,%s,964982703\n" % row)
    assert collab.main([str(path), "--implicit", "--alpha", "1.0"]) == 0
    out = capsys.readouterr().out
    assert "precisionAt(10) = %r" % g["precision_at_k"] in out
    assert "ndcgAt(10) = %r" % g["ndcg_at_k"] in out
    assert "meanAveragePrecision = %r" % g["mean_average_precision"] in out
    assert "Root-mean-square error" not in out
    for title in ("itemFactors", "userFactors", "userRecs", "movieRecs", "userSubsetRecs", "movieSubSetRecs"):
        assert title in out
    tr, te = collab.random_split(len(fixture["userId"]), (0.8, 0.2), 0)
    model = collab.als({k: v[tr] for k, v in fixture.items()}, implicit_prefs=True, alpha=1.0)
    assert len(tr) == g["n_train"] and len(model.user_ids) == g["n_users"] and len(model.item_ids) == g["n_movies"]
    assert model.user_factors[:3].astype(np.float64).tolist() == g["user_factors_head"]
    assert model.item_factors[:3].astype(np.float64).tolist() == g["item_factors_head"]
    users, _, (off, _) = model.ranking_queries({k: v[te] for k, v in fixture.items()})
    assert len(users) == g["n_queries"] and int(off[-1]) == g["n_relevant"]
    _, ids, sc = model.recommend_for_all_users(10)
    assert ids[:3].tolist() == g["user_recs_head"]["ids"]
    assert sc[:3].astype(np.float64).tolist() == g["user_recs_head"]["scores"]
    _, ids, sc = model.recommend_for_all_items(10)
    assert ids[:3].tolist() == g["movie_recs_head"]["ids"]
    assert collab.main([str(path), "--implicit", "--cv"]) == 2     # CrossValidator has no ranking evaluator
    assert collab.main([str(path), "--alpha", "2"]) == 2
