"""ALS and its recommendations on the device (`collab`, csrc/als.cu) against the C oracle, bit for bit."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import als_cext as X
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import collab
from sparrowrecsys_b200.model import launch_count

from test_als_oracle import (GOLDEN, _raw_fit, _raw_recommend, bits, fixture_ratings, hand_cases, same_fit,
                             singular_case)

pytestmark = pytest.mark.gpu


def _dev(r, **kw):
    m = collab.als(r, **kw)
    return m.user_ids, m.user_factors, m.item_ids, m.item_factors


def _check(u, m, r, **kw):
    dev = _dev({"userId": u, "movieId": m, "rating": r}, **kw)
    same_fit(dev, X.fit(u, m, np.asarray(r, np.float32), **kw))
    return dev


@pytest.fixture(scope="module")
def fixture():
    return fixture_ratings()


@pytest.fixture(scope="module")
def script_models(fixture):
    out = {}
    for seed in (0, 1):
        tr, _ = collab.random_split(len(fixture["userId"]), (0.8, 0.2), seed)
        sub = {k: v[tr] for k, v in fixture.items()}
        out[seed] = (sub, collab.als(sub, rank=10, max_iter=5, reg_param=0.01, seed=seed))
    return out


@pytest.mark.parametrize("seed", [0, 1])
def test_the_scripts_fit_is_bit_equal_to_the_c_oracle(script_models, seed):
    sub, model = script_models[seed]
    ref = X.fit(sub["userId"], sub["movieId"], sub["rating"], rank=10, max_iter=5, reg_param=0.01, seed=seed)
    same_fit((model.user_ids, model.user_factors, model.item_ids, model.item_factors), ref)


@pytest.mark.parametrize("rank", [1, 16, 32, 33, 64])
@pytest.mark.parametrize("max_iter", [1, 2])
def test_ranks_and_iterations_bit_equal_to_the_c_oracle(fixture, rank, max_iter):
    _check(fixture["userId"], fixture["movieId"], fixture["rating"], rank=rank, max_iter=max_iter,
           reg_param=0.01, seed=rank)


@pytest.mark.parametrize("name", sorted(hand_cases()))
@pytest.mark.parametrize("rank", [1, 10, 33, 64])
def test_hand_built_cases_bit_equal_to_the_c_oracle(name, rank):
    u, m, r = hand_cases()[name]
    _check(u, m, r, rank=rank, max_iter=2, reg_param=0.05, seed=rank)


def test_repeat_runs_give_the_same_bits(fixture):
    a = _dev(fixture, rank=12, max_iter=2, seed=5)
    same_fit(a, _dev(fixture, rank=12, max_iter=2, seed=5))


def test_a_singular_system_names_the_entity_and_writes_nothing():
    u, m, r = singular_case()
    lib = _lib.load()
    u32, m32, r32 = (np.ascontiguousarray(x, t) for x, t in ((u, np.int32), (m, np.int32), (r, np.float32)))
    p = _lib.SrsAlsParams(2, 1, 0.0, 0)
    ui, mi = np.full(8, -7, np.int32), np.full(8, -7, np.int32)
    uf, mf = np.full((8, 2), 3.5, np.float32), np.full((8, 2), 3.5, np.float32)
    nu, nm = C.c_int32(-1), C.c_int32(-1)
    rc = lib.srs_als_fit_host(u32.ctypes.data, m32.ctypes.data, r32.ctypes.data, len(u32), C.byref(p), 0, 8, 8,
                              ui.ctypes.data, uf.ctypes.data, C.byref(nu), mi.ctypes.data, mf.ctypes.data,
                              C.byref(nm))
    assert rc == _lib.SRS_ERR_INVALID
    msg = lib.srs_last_error().decode()
    assert "user 9" in msg and "iteration 1" in msg, msg
    assert nu.value == 0 and nm.value == 0
    assert np.all(ui == -7) and np.all(mi == -7) and np.all(uf == 3.5) and np.all(mf == 3.5)
    with pytest.raises(ValueError, match="user 9"):
        collab.als({"userId": u, "movieId": m, "rating": r}, rank=2, max_iter=1, reg_param=0.0)
    _check(u, m, r, rank=2, max_iter=1, reg_param=0.01, seed=0)


def test_too_little_capacity_is_a_range_error():
    u, m, r = hand_cases()["one_rating_user"]
    assert _raw_fit(u, m, r, cap=5) == (_lib.SRS_ERR_RANGE, 0, 0)


def test_rejections_launch_nothing():
    n0 = launch_count()
    assert _raw_fit([1, 2], [3, 4], [4.0, 5.0], rank=0)[0] == _lib.SRS_ERR_INVALID
    assert _raw_fit([1, 2], [3, -4], [4.0, 5.0])[0] == _lib.SRS_ERR_INVALID
    assert _raw_recommend(np.ones((2, 3)), [1, 2, 2, 4], np.ones((4, 3)), 3, 5) == _lib.SRS_ERR_INVALID
    assert _raw_recommend(np.ones((2, 3)), [1, 2, 3, 4], np.ones((4, 3)), 3, 200) == _lib.SRS_ERR_INVALID
    assert launch_count() == n0


def _same_recs(dev, ref):
    assert np.array_equal(dev[0], ref[0]), (dev[0][:2], ref[0][:2])
    assert np.array_equal(bits(dev[1]), bits(ref[1]))


@pytest.mark.parametrize("num", [1, 10, 128])
def test_recommend_for_all_bit_equal_to_the_c_oracle(script_models, num):
    _, model = script_models[0]
    uids, ids, sc = model.recommend_for_all_users(num)
    assert np.array_equal(uids, model.user_ids) and ids.shape == (len(uids), num)
    _same_recs((ids, sc), X.recommend(model.user_factors, model.item_ids, model.item_factors, num))
    mids, ids, sc = model.recommend_for_all_items(num)
    assert np.array_equal(mids, model.item_ids)
    _same_recs((ids, sc), X.recommend(model.item_factors, model.user_ids, model.user_factors, num))


def test_num_beyond_the_destinations_returns_them_all():
    rng = np.random.default_rng(4)
    src = rng.normal(size=(70, 9)).astype(np.float32)
    dst = rng.normal(size=(37, 9)).astype(np.float32)
    ids = np.sort(rng.choice(10 ** 6, 37, replace=False)).astype(np.int32)
    for num in (37, 38, 128):
        got = collab.recommend(src, ids, dst, num)
        assert got[0].shape == (70, 37)
        _same_recs(got, X.recommend(src, ids, dst, num))


def test_subsets_match_the_c_oracle(script_models):
    _, model = script_models[1]
    want_u = np.array([model.user_ids[5], model.user_ids[0], 10 ** 9, model.user_ids[5]])
    su, ids, sc = model.recommend_for_user_subset(want_u, 10)
    assert su.tolist() == sorted({int(model.user_ids[0]), int(model.user_ids[5])})
    _same_recs((ids, sc), X.recommend(model.user_factors[[0, 5]], model.item_ids, model.item_factors, 10))
    sm, ids, sc = model.recommend_for_item_subset([model.item_ids[-1], -3], 7)
    assert sm.tolist() == [int(model.item_ids[-1])]
    _same_recs((ids, sc), X.recommend(model.item_factors[-1:], model.user_ids, model.user_factors, 7))


@pytest.mark.parametrize("num", [1, 3, 10, 128])
def test_planted_ties_go_to_the_lower_id(num):
    rng = np.random.default_rng(9)
    n_dst, k = 700, 33
    dst = rng.normal(size=(n_dst, k)).astype(np.float32)
    for a, b in ((3, 600), (3, 129), (3, 140), (250, 10), (699, 0)):
        dst[b] = dst[a]                                    # equal rows across tiles: equal scores for every source
    src = rng.normal(size=(101, k)).astype(np.float32)
    src[7] = 0                                             # all scores 0 for one source
    src[8] = -dst[3]
    ids = np.arange(n_dst, dtype=np.int32) * 3 + 1
    got = collab.recommend(src, ids, dst, num)
    _same_recs(got, X.recommend(src, ids, dst, num))
    assert got[0][7].tolist() == ids[:min(num, n_dst)].tolist()


def test_the_scripts_sequence_gives_the_recorded_rmse(fixture, script_models):
    with open(os.path.join(GOLDEN, "als_fit.json")) as f:
        rec = json.load(f)
    for seed in (0, 1):
        sub, model = script_models[seed]
        g = rec["seeds"][str(seed)]
        _, te = collab.random_split(len(fixture["userId"]), (0.8, 0.2), seed)
        test = {k: v[te] for k, v in fixture.items()}
        kept, pred = model.transform(test)
        assert len(sub["userId"]) == g["n_train"] and len(kept) == g["n_kept"]
        assert int(np.sum(kept.astype(np.int64) * (np.arange(len(kept)) % 7 + 1))) == g["kept_checksum"]
        assert collab.rmse(test["rating"][kept], pred) == g["rmse"]
        _, ids, sc = model.recommend_for_all_users(10)
        assert ids[:3].tolist() == g["user_recs_head"]["ids"]
        assert sc[:3].astype(np.float64).tolist() == g["user_recs_head"]["scores"]
        _, ids, sc = model.recommend_for_all_items(10)
        assert ids[:3].tolist() == g["movie_recs_head"]["ids"]


def test_the_command_prints_the_scripts_output(tmp_path, capsys):
    r = fixture_ratings()
    path = tmp_path / "ratings.csv"
    n = 30000
    with open(path, "w") as f:
        f.write("userId,movieId,rating,timestamp\n")
        for row in zip(r["userId"][:n].tolist(), r["movieId"][:n].tolist(), r["rating"][:n].tolist()):
            f.write("%d,%d,%s,964982703\n" % row)
    assert collab.main([str(path)]) == 0
    out = capsys.readouterr().out
    tr, te = collab.random_split(n, (0.8, 0.2), 0)
    sub = {k: v[:n] for k, v in r.items()}
    model = collab.als({k: v[tr] for k, v in sub.items()})
    kept, pred = model.transform({k: v[te] for k, v in sub.items()})
    assert "Root-mean-square error = %r" % collab.rmse(sub["rating"][te][kept], pred) in out
    for title in ("itemFactors", "userFactors", "userRecs", "movieRecs", "userSubsetRecs", "movieSubSetRecs"):
        assert title in out
