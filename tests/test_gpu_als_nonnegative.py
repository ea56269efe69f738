"""Nonnegative ALS on the device (`collab`, csrc/als.cu's NNLS tail) against the C oracle, bit for bit: single
explicit and implicit fits, the batched fit with mixed solvers, and the script's `--nonnegative` commands."""
import json
import math
import os

import numpy as np
import pytest

from oracle import als_nnls_cext as XN
from sparrowrecsys_b200 import collab

from test_als_nonnegative_oracle import chunk_edge_case, nnls_cases
from test_als_implicit_oracle import implicit_cases
from test_als_oracle import GOLDEN, fixture_ratings, same_fit

pytestmark = pytest.mark.gpu


def _dev(r, **kw):
    m = collab.als(r, nonnegative=True, **kw)
    return m.user_ids, m.user_factors, m.item_ids, m.item_factors


def _check(u, m, r, **kw):
    dev = _dev({"userId": u, "movieId": m, "rating": r}, **kw)
    same_fit(dev, XN.fit(u, m, np.asarray(r, np.float32), **kw))
    assert np.all(dev[1] >= 0) and np.all(dev[3] >= 0)
    return dev


@pytest.fixture(scope="module")
def fixture():
    return fixture_ratings()


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("implicit", [False, True])
def test_the_scripts_fit_is_bit_equal_to_the_c_oracle(fixture, seed, implicit):
    tr, _ = collab.random_split(len(fixture["userId"]), (0.8, 0.2), seed)
    sub = {k: v[tr] for k, v in fixture.items()}
    _check(sub["userId"], sub["movieId"], sub["rating"], rank=10, max_iter=5, reg_param=0.01, seed=seed,
           implicit_prefs=implicit, alpha=1.0)


@pytest.mark.parametrize("rank", [1, 16, 32, 33, 64])
@pytest.mark.parametrize("max_iter", [1, 2])
@pytest.mark.parametrize("implicit", [False, True])
def test_ranks_and_iterations_bit_equal_to_the_c_oracle(fixture, rank, max_iter, implicit):
    _check(fixture["userId"], fixture["movieId"], fixture["rating"], rank=rank, max_iter=max_iter, reg_param=0.01,
           seed=rank, implicit_prefs=implicit, alpha=1.0)


@pytest.mark.parametrize("name", sorted(nnls_cases()))
@pytest.mark.parametrize("rank", [1, 10, 33, 64])
def test_hand_built_cases_bit_equal_to_the_c_oracle(name, rank):
    u, m, r, reg = nnls_cases()[name]
    _check(u, m, r, rank=rank, max_iter=2, reg_param=reg, seed=rank)


@pytest.mark.parametrize("name", sorted(implicit_cases()))
@pytest.mark.parametrize("alpha", [0.0, 1.0, 40.0])
def test_implicit_hand_built_cases_bit_equal_to_the_c_oracle(name, alpha):
    u, m, r = implicit_cases()[name]
    _check(u, m, r, rank=10, max_iter=2, reg_param=0.05, seed=3, implicit_prefs=True, alpha=alpha)


def test_the_ill_conditioned_case_reaches_iter_max_on_the_device_too():
    u, m, r, reg = nnls_cases()["ill_conditioned"]
    _check(u, m, r, rank=64, max_iter=1, reg_param=reg, seed=0)


def test_entities_at_the_chunk_edges(fixture):
    u, m, r = chunk_edge_case()
    for rank in (10, 64):
        _check(u, m, r, rank=rank, max_iter=2, reg_param=0.01, seed=1)
        _check(u, m, r, rank=rank, max_iter=2, reg_param=0.01, seed=1, implicit_prefs=True, alpha=1.0)


def test_regparam_zero_with_an_all_zero_system_is_not_an_error():
    u, m, r, _ = nnls_cases()["all_zero_system"]
    uids, U, _, _ = _check(u, m, r, rank=2, max_iter=1, reg_param=0.0, seed=0)
    assert np.all(U[np.searchsorted(uids, 9)] == 0)
    with pytest.raises(ValueError, match="singular"):
        collab.als({"userId": u, "movieId": m, "rating": r}, rank=2, max_iter=1, reg_param=0.0)


def test_repeat_runs_give_the_same_bits(fixture):
    a = _dev(fixture, rank=12, max_iter=2, seed=5)
    same_fit(a, _dev(fixture, rank=12, max_iter=2, seed=5))
    a = _dev(fixture, rank=12, max_iter=2, seed=5, implicit_prefs=True, alpha=3.0)
    same_fit(a, _dev(fixture, rank=12, max_iter=2, seed=5, implicit_prefs=True, alpha=3.0))


def test_the_default_call_is_unchanged(fixture):
    for kw in ({}, {"implicit_prefs": True, "alpha": 2.0}):
        a = collab.als(fixture, rank=6, max_iter=2, seed=3, **kw)
        b = collab.als(fixture, rank=6, max_iter=2, seed=3, nonnegative=False, **kw)
        same_fit((a.user_ids, a.user_factors, a.item_ids, a.item_factors),
                 (b.user_ids, b.user_factors, b.item_ids, b.item_factors))


# ---- the batched fit ----------------------------------------------------------------------------------------------
GRID = [("nonnegative", [False, True]), ("reg_param", [0.01, 0.1])]


def test_a_mixed_batch_gives_each_model_its_single_fits_bits(fixture):
    n = len(fixture["userId"])
    fold = collab.fold_ids(n, 3, 0)
    points = [dict(dict(rank=8, max_iter=2, reg_param=0.01), **pm) for pm in collab.param_maps(GRID)]
    specs = [dict(p, exclude_fold=f) for f in range(3) for p in points]
    specs.append(dict(rank=5, max_iter=1, reg_param=0.05, exclude_fold=-1, nonnegative=True))
    models = collab.als_folds(fixture, fold, 3, specs, seed=2)
    for spec, got in zip(specs, models):
        rows = fold != spec["exclude_fold"]
        want = collab.als({k: v[rows] for k, v in fixture.items()}, rank=spec["rank"], max_iter=spec["max_iter"],
                          reg_param=spec["reg_param"], seed=2, nonnegative=spec.get("nonnegative", False))
        same_fit((got.user_ids, got.user_factors, got.item_ids, got.item_factors),
                 (want.user_ids, want.user_factors, want.item_ids, want.item_factors))
        if spec.get("nonnegative"):
            assert np.all(got.user_factors >= 0) and np.all(got.item_factors >= 0)
    # the Cholesky models keep srs_als_fit_folds_host's bits
    plain = [s for s in specs if not s.get("nonnegative")]
    for a, b in zip(collab.als_folds(fixture, fold, 3, plain, seed=2), [m for s, m in zip(specs, models)
                                                                          if not s.get("nonnegative")]):
        same_fit((a.user_ids, a.user_factors, a.item_ids, a.item_factors),
                 (b.user_ids, b.user_factors, b.item_ids, b.item_factors))


def test_cross_validate_refits_the_best_point_with_its_flag(fixture):
    tr, te = collab.random_split(len(fixture["userId"]), (0.8, 0.2), 0)
    test = {k: v[te] for k, v in fixture.items()}
    res = collab.cross_validate(test, GRID, num_folds=3, cold_start_strategy="drop", rank=6, max_iter=2)
    assert [p["nonnegative"] for p in res.param_maps] == [False, True, False, True]
    best = res.param_maps[res.best_index]
    want = collab.als(test, rank=6, max_iter=2, reg_param=best["reg_param"], nonnegative=best["nonnegative"])
    same_fit((res.best_model.user_ids, res.best_model.user_factors, res.best_model.item_ids,
              res.best_model.item_factors), (want.user_ids, want.user_factors, want.item_ids, want.item_factors))
    for flag in (False, True):                               # the estimator default, refit included
        res = collab.cross_validate(test, [("reg_param", [0.01, 0.1])], num_folds=3, cold_start_strategy="drop",
                                    rank=6, max_iter=2, nonnegative=flag)
        best = res.param_maps[res.best_index]
        assert best.get("nonnegative", False) == flag
        want = collab.als(test, rank=6, max_iter=2, reg_param=best["reg_param"], nonnegative=flag)
        same_fit((res.best_model.user_ids, res.best_model.user_factors), (want.user_ids, want.user_factors))


def test_a_call_without_the_setting_keeps_todays_result(fixture):
    tr, te = collab.random_split(len(fixture["userId"]), (0.8, 0.2), 0)
    test = {k: v[te] for k, v in fixture.items()}
    res = collab.cross_validate(test, [("reg_param", [0.01, 0.1])], num_folds=3, cold_start_strategy="drop",
                                rank=6, max_iter=2)
    assert res.param_maps == [dict(rank=6, max_iter=2, reg_param=0.01), dict(rank=6, max_iter=2, reg_param=0.1)]
    assert "nonnegative" not in res.best_params


# ---- the script's --nonnegative commands --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ratings_csv(tmp_path_factory, fixture):
    path = tmp_path_factory.mktemp("nnls") / "ratings.csv"
    with open(path, "w") as f:
        f.write("userId,movieId,rating,timestamp\n")
        for row in zip(fixture["userId"].tolist(), fixture["movieId"].tolist(), fixture["rating"].tolist()):
            f.write("%d,%d,%s,964982703\n" % row)
    with open(os.path.join(GOLDEN, "als_nonnegative.json")) as f:
        return str(path), json.load(f)


def _factor_lines(out, title, head):
    lines = out.splitlines()
    at = lines.index(title)
    for i, row in enumerate(head):
        assert lines[at + 1 + i].split("\t")[1] == "[%s]" % ", ".join(repr(float(v)) for v in row)


def _rec_lines(out, title, rec):
    lines = out.splitlines()
    at = lines.index(title)
    for i, who in enumerate(rec["users"] if "users" in rec else rec["movies"]):
        want = "%d\t[%s]" % (who, ", ".join("[%d, %s]" % (a, repr(float(b)))
                                            for a, b in zip(rec["ids"][i], rec["scores"][i])))
        assert lines[at + 1 + i] == want


def test_the_nonnegative_command_prints_the_recorded_output(ratings_csv, capsys):
    path, g = ratings_csv
    assert collab.main([path, "--nonnegative"]) == 0
    out = capsys.readouterr().out
    e = g["explicit"]
    assert "Root-mean-square error = %r" % e["rmse"] in out
    _factor_lines(out, "itemFactors", e["item_factors_head"])
    _factor_lines(out, "userFactors", e["user_factors_head"])
    _rec_lines(out, "userRecs", e["user_recs_head"])
    _rec_lines(out, "movieRecs", e["movie_recs_head"])


def test_the_nonnegative_implicit_command_prints_the_recorded_output(ratings_csv, capsys):
    path, g = ratings_csv
    assert collab.main([path, "--nonnegative", "--implicit", "--alpha", "1.0"]) == 0
    out = capsys.readouterr().out
    i = g["implicit"]
    assert "precisionAt(10) = %r" % i["precision_at_k"] in out
    assert "ndcgAt(10) = %r" % i["ndcg_at_k"] in out
    assert "meanAveragePrecision = %r" % i["mean_average_precision"] in out
    assert "Root-mean-square error" not in out
    _factor_lines(out, "itemFactors", i["item_factors_head"])
    _factor_lines(out, "userFactors", i["user_factors_head"])
    _rec_lines(out, "userRecs", i["user_recs_head"])
    _rec_lines(out, "movieRecs", i["movie_recs_head"])


def test_the_nonnegative_cv_command_prints_the_recorded_output(ratings_csv, capsys):
    path, g = ratings_csv
    assert collab.main([path, "--nonnegative", "--cv"]) == 0
    out = capsys.readouterr().out
    assert "Root-mean-square error = %r" % g["explicit"]["rmse"] in out
    avg = g["cv"]["avg_metrics"]
    assert "avgMetrics = %r" % avg in out or (all(math.isnan(v) for v in avg) and "avgMetrics = [nan]" in out)
    assert "cold validation rows per fold = %r" % g["cv"]["cold_rows"] in out
    assert collab.main([path, "--nonnegative", "--implicit", "--cv"]) == 2
    assert collab.main([path, "--nonnegative", "--alpha", "2"]) == 2
