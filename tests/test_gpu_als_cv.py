"""The batched ALS fit (`collab.als_folds`, `srs_als_fit_folds_host`) against one `collab.als` per model, and
`collab.cross_validate` against the C oracle, bit for bit."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

from oracle import als_cv as O
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import collab
from sparrowrecsys_b200.model import launch_count

from test_als_oracle import GOLDEN, fixture_ratings, same_fit, singular_case

pytestmark = pytest.mark.gpu

POINTS = [dict(rank=k, reg_param=reg, max_iter=it) for k in (1, 10, 33, 64) for reg in (0.01, 0.1) for it in (1, 2)]


@pytest.fixture(scope="module")
def fixture():
    return fixture_ratings()


def _same_as_single_fits(ratings, fold, models, got, seed):
    for spec, model in zip(models, got):
        rows = fold != spec["exclude_fold"]
        sub = {c: v[rows] for c, v in ratings.items()}
        ref = collab.als(sub, rank=spec["rank"], max_iter=spec["max_iter"], reg_param=spec["reg_param"], seed=seed)
        same_fit((model.user_ids, model.user_factors, model.item_ids, model.item_factors),
                 (ref.user_ids, ref.user_factors, ref.item_ids, ref.item_factors))


@pytest.mark.parametrize("k", [2, 3, 10])
def test_every_model_equals_its_single_fit(fixture, k):
    fold = collab.fold_ids(len(fixture["userId"]), k, seed=k)
    if k < 10:                                             # the whole grid for every fold
        models = [dict(p, exclude_fold=f) for f in range(k) for p in POINTS]
    else:                                                  # each fold with four of the grid's points
        models = [dict(POINTS[(4 * f + j) % len(POINTS)], exclude_fold=f) for f in range(k) for j in range(4)]
    models.append(dict(rank=10, reg_param=0.01, max_iter=2, exclude_fold=-1))
    assert len(models) <= 64
    got = collab.als_folds(fixture, fold, k, models, seed=11)
    assert len(got) == len(models)
    _same_as_single_fits(fixture, fold, models, got, 11)


def test_repeat_runs_give_the_same_bits(fixture):
    fold = collab.fold_ids(len(fixture["userId"]), 3, seed=1)
    models = [dict(POINTS[i], exclude_fold=i % 3) for i in (3, 8, 13)]
    a = collab.als_folds(fixture, fold, 3, models, seed=2)
    b = collab.als_folds(fixture, fold, 3, models, seed=2)
    for x, y in zip(a, b):
        same_fit((x.user_ids, x.user_factors, x.item_ids, x.item_factors),
                 (y.user_ids, y.user_factors, y.item_ids, y.item_factors))


def test_launches_per_half_step_do_not_depend_on_the_model_count(fixture):
    fold = collab.fold_ids(len(fixture["userId"]), 5, seed=0)
    counts = {}
    for M in (1, 7):
        for it in (1, 2):
            models = [dict(rank=4 + i, reg_param=0.05, max_iter=1 + (i % it), exclude_fold=i % 5) for i in range(M)]
            models[0]["max_iter"] = it
            n0 = launch_count()
            collab.als_folds(fixture, fold, 5, models)
            counts[M, it] = launch_count() - n0
    assert counts[1, 1] == counts[7, 1] and counts[1, 2] == counts[7, 2]
    assert counts[1, 2] - counts[1, 1] == 2                # one launch per half-step


def test_a_singular_model_is_named_and_nothing_is_written():
    u, m, r = singular_case()                              # rank 2, reg 0: user 9's system is all zero
    u, m, r = np.r_[u, u[4:]], np.r_[m, m[4:]], np.r_[r, r[4:]]
    n = len(u)
    fold = np.r_[np.zeros(n - (n - 4) // 2), np.ones((n - 4) // 2)].astype(np.int32)   # fold 0: the singular case
    models = [(2, 1, 0.01, -1), (2, 1, 0.0, 1), (2, 1, 0.0, 1), (2, 1, 0.01, 0)]
    lib = _lib.load()
    u32, m32, r32 = (np.ascontiguousarray(x, t) for x, t in ((u, np.int32), (m, np.int32), (r, np.float32)))
    specs = (_lib.SrsAlsModel * 4)(*[_lib.SrsAlsModel(*p) for p in models])
    ui, mi = np.full(4 * 8, -7, np.int32), np.full(4 * 8, -7, np.int32)
    uf, mf = np.full(4 * 8 * 2, 3.5, np.float32), np.full(4 * 8 * 2, 3.5, np.float32)
    nu, nm = np.full(4, -1, np.int32), np.full(4, -1, np.int32)
    rc = lib.srs_als_fit_folds_host(u32.ctypes.data, m32.ctypes.data, r32.ctypes.data, fold.ctypes.data, n, 2, specs,
                                    4, 0, 0, 8, 8, ui.ctypes.data, uf.ctypes.data, nu.ctypes.data, mi.ctypes.data,
                                    mf.ctypes.data, nm.ctypes.data)
    assert rc == _lib.SRS_ERR_INVALID
    msg = lib.srs_last_error().decode()
    assert "model 1:" in msg and "user 9" in msg and "iteration 1" in msg, msg
    assert np.all(nu == 0) and np.all(nm == 0)
    assert np.all(ui == -7) and np.all(mi == -7) and np.all(uf == 3.5) and np.all(mf == 3.5)
    ratings = {"userId": u, "movieId": m, "rating": r}
    keep = [dict(rank=2, max_iter=1, reg_param=p[2], exclude_fold=p[3]) for p in (models[0], models[3])]
    _same_as_single_fits(ratings, fold, keep, collab.als_folds(ratings, fold, 2, keep), 0)


@pytest.fixture(scope="module")
def script_test():
    r = fixture_ratings()
    _, te = collab.random_split(len(r["userId"]), (0.8, 0.2), 0)
    return {k: v[te] for k, v in r.items()}


@pytest.mark.parametrize("metric,strategy", [("rmse", "nan"), ("rmse", "drop"), ("mse", "drop"), ("mae", "drop")])
def test_cross_validation_equals_the_c_oracle(script_test, metric, strategy):
    grid = [("reg_param", [0.01, 0.1]), ("rank", [4])]
    kw = dict(num_folds=4, metric=metric, cold_start_strategy=strategy, seed=5, max_iter=3, als_seed=6)
    got = collab.cross_validate(script_test, grid, **kw)
    ref = O.cross_validate(script_test, grid, **kw)
    assert repr(got.fold_metrics) == repr(ref["fold_metrics"])
    assert repr(got.avg_metrics) == repr(ref["avg_metrics"])
    assert got.best_index == ref["best_index"] and got.cold_rows == ref["cold_rows"]
    assert got.param_maps == ref["param_maps"] and got.best_params == ref["param_maps"][got.best_index]
    best = collab.als(script_test, seed=6, **got.best_params)
    same_fit((got.best_model.user_ids, got.best_model.user_factors, got.best_model.item_ids,
              got.best_model.item_factors), (best.user_ids, best.user_factors, best.item_ids, best.item_factors))


def test_more_models_than_one_batch_holds(script_test):
    grid = [("rank", [2, 3, 4, 5, 6, 7, 8]), ("max_iter", [1])]            # 10 folds x 7 points: two batches
    got = collab.cross_validate(script_test, grid, num_folds=10, cold_start_strategy="drop")
    ref = O.cross_validate(script_test, grid, num_folds=10, cold_start_strategy="drop")
    assert repr(got.fold_metrics) == repr(ref["fold_metrics"])


def test_the_scripts_cv_step_gives_the_recorded_metrics(tmp_path, capsys, script_test):
    with open(os.path.join(GOLDEN, "als_cv.json")) as f:
        rec = json.load(f)
    assert len(script_test["userId"]) == rec["n_rows"]
    for strategy in ("nan", "drop"):
        res = collab.cross_validate(script_test, [("reg_param", [0.01])], num_folds=10, cold_start_strategy=strategy)
        assert repr(res.fold_metrics) == repr(rec[strategy]["fold_metrics"])
        assert repr(res.avg_metrics) == repr(rec[strategy]["avg_metrics"])
        assert res.cold_rows == rec["cold_rows"]
    assert math.isnan(rec["nan"]["avg_metrics"][0]) and all(c > 0 for c in rec["cold_rows"])
    r = fixture_ratings()
    path = tmp_path / "ratings.csv"
    with open(path, "w") as f:
        f.write("userId,movieId,rating,timestamp\n")
        for row in zip(r["userId"].tolist(), r["movieId"].tolist(), r["rating"].tolist()):
            f.write("%d,%d,%s,964982703\n" % row)
    assert collab.main([str(path), "--cv"]) == 0
    out = capsys.readouterr().out
    assert "avgMetrics = [nan]\n" in out
    assert "cold validation rows per fold = %r\n" % rec["cold_rows"] in out
    assert collab.main([str(path)]) == 0
    assert "avgMetrics" not in capsys.readouterr().out
