"""Cross-validating ALS (`collab.cross_validate`, oracle/als_cv.py): the host-side rules and the batched ABI's
device-free rejections.  DESIGN.md section 4.15 gives the semantics."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import als as A
from oracle import als_cext as X
from oracle import als_cv as O
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import collab
from sparrowrecsys_b200.model import launch_count

from test_als_oracle import bits, hand_cases

NAN = float("nan")


# ---- folds ------------------------------------------------------------------------------------------------------
def test_fold_bounds_are_float32_quotients_widened_to_double():
    f01 = float(np.float32(0.1))                           # 0.10000000149...: fold 1's upper bound
    assert f01 > 0.1
    u = np.array([0.1, np.nextafter(0.1, 1.0), np.nextafter(f01, 0.0), f01, 0.0, np.nextafter(1.0, 0.0)])
    assert collab._fold_of(u, 10).tolist() == [0, 0, 0, 1, 0, 9]


@pytest.mark.parametrize("k", [2, 3, 10])
def test_folds_partition_the_rows_and_training_is_the_complement(k):
    n, seed = 4000, 3
    pairs = collab.k_fold(n, k, seed)
    assert len(pairs) == k
    seen = np.zeros(n, np.int64)
    for tr, va in pairs:
        assert np.all(np.diff(tr) > 0) and np.all(np.diff(va) > 0)          # input order
        assert np.array_equal(np.sort(np.r_[tr, va]), np.arange(n))
        seen[va] += 1
    assert np.all(seen == 1)
    fold = collab.fold_ids(n, k, seed)
    assert np.array_equal(fold, O.fold_of(n, k, seed))
    u = collab._uniforms(seed, n)                          # one draw per row, shared by every fold
    for f, (_, va) in enumerate(pairs):
        lb, ub = float(np.float32(f) / np.float32(k)), float(np.float32(f + 1) / np.float32(k))
        assert np.array_equal(va, np.flatnonzero((u >= lb) & (u < ub)))


def test_fewer_than_two_folds_is_an_error():
    for k in (0, 1):
        with pytest.raises(ValueError, match="num_folds"):
            collab.k_fold(10, k)
        with pytest.raises(ValueError, match="num_folds"):
            collab.cross_validate({"userId": [1], "movieId": [2], "rating": [3.0]}, [("reg_param", [0.1])], k)


# ---- grid, averages, best point ---------------------------------------------------------------------------------
def test_grid_order_first_param_fastest():
    pairs = [("rank", [1, 2]), ("reg_param", [0.1, 0.2, 0.3]), ("max_iter", [4])]
    maps = collab.param_maps(pairs)
    assert [(m["rank"], m["reg_param"]) for m in maps] == [(1, 0.1), (2, 0.1), (1, 0.2), (2, 0.2), (1, 0.3), (2, 0.3)]
    assert all(m["max_iter"] == 4 for m in maps)
    assert maps == O.grid(pairs) == collab.param_maps(dict(pairs))
    assert collab.param_maps([]) == [{}]                   # no params: one map of the estimator's values


def test_bad_grids_are_errors():
    for grid in ([("reg_param", [])], [("alpha", [1.0])], [("rank", [1]), ("rank", [2])]):
        with pytest.raises(ValueError):
            collab.param_maps(grid)
    with pytest.raises(ValueError, match="empty"):
        collab.cross_validate({"userId": [1], "movieId": [2], "rating": [3.0]}, [("rank", [])])


def test_averages_sum_in_fold_order():
    fm = [[1e16, 1.0], [1.0, 2.0], [-1e16, 4.0]]
    assert collab.average_metrics(fm) == [((1e16 + 1.0) - 1e16) / 3, (1.0 + 2.0 + 4.0) / 3] == [0.0, 7.0 / 3]
    assert math.isnan(collab.average_metrics([[1.0], [NAN]])[0])


@pytest.mark.parametrize("metrics,want", [([NAN, 2.0, 1.0, 1.0], 2), ([NAN, NAN], 0), ([1.0, NAN, 1.0], 0),
                                          ([3.0, 0.5, NAN, 0.5, 0.25], 4), ([0.0, -0.0], 1), ([7.0], 0)])
def test_best_index_is_min_by_double_compare(metrics, want):
    assert collab.best_index(metrics) == want


# ---- cold rows, metrics -----------------------------------------------------------------------------------------
def _hand_model():
    rng = np.random.default_rng(1)
    uf = rng.normal(size=(3, 5)).astype(np.float32)
    mf = rng.normal(size=(4, 5)).astype(np.float32)
    return collab.AlsModel(np.array([2, 5, 9], np.int32), uf, np.array([1, 3, 4, 8], np.int32), mf)


def test_nan_cold_rows_give_a_nan_rmse_and_drop_a_finite_one():
    model = _hand_model()
    test = {"userId": np.array([5, 6, 2, 9, 9, 1]), "movieId": np.array([3, 3, 8, 2, 1, 1]),
            "rating": np.array([4.0, 3.0, 2.5, 1.0, 5.0, 3.5], np.float32)}
    rows, pred = model.transform(test, cold_start_strategy="nan")
    assert rows.tolist() == list(range(6))
    assert np.isnan(pred).tolist() == [False, True, False, True, False, True]
    kept, kp = model.transform(test)
    assert kept.tolist() == [0, 2, 4] and np.array_equal(bits(pred[kept]), bits(kp))
    assert model.cold_rows(test) == 3
    assert math.isnan(collab.rmse(test["rating"], pred))
    assert math.isfinite(collab.rmse(test["rating"][kept], kp))
    uids, uf, mids, mf = model.user_ids, model.user_factors, model.item_ids, model.item_factors
    for strategy, (r, p) in (("nan", (rows, pred)), ("drop", (kept, kp))):
        lab, op, cold = O.transform((uids, uf, mids, mf), test, strategy)
        assert cold == 3 and np.array_equal(lab, test["rating"][r]) and np.array_equal(bits(op), bits(p))
    with pytest.raises(ValueError):
        model.transform(test, cold_start_strategy="error")


def test_mse_and_mae_against_hand_sums():
    lab = np.array([4.0, 3.5, 1.0, 2.0], np.float32)
    pred = np.array([3.9, 3.0, 2.5, 2.25], np.float32)
    d = [float(a) - float(b) for a, b in zip(lab, pred)]
    ss = ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) + d[3] * d[3]
    norm = math.sqrt(ss)
    assert collab.mse(lab, pred) == norm * norm / 4 == O.metric_value("mse", lab, pred)
    assert collab.mae(lab, pred) == (((abs(d[0]) + abs(d[1])) + abs(d[2])) + abs(d[3])) / 4 \
        == O.metric_value("mae", lab, pred)
    assert collab.rmse(lab, pred) == math.sqrt(norm * norm / 4) == O.metric_value("rmse", lab, pred)
    assert all(math.isnan(f([], [])) for f in (collab.mse, collab.mae, collab.rmse))


# ---- the oracle -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric,strategy", [("rmse", "nan"), ("rmse", "drop"), ("mae", "drop")])
def test_oracle_cross_validation_equals_a_hand_loop_of_the_oracle_fit(metric, strategy):
    u, m, r = hand_cases()["one_rating_user"]
    ratings = {"userId": np.asarray(u, np.int32), "movieId": np.asarray(m, np.int32),
               "rating": np.asarray(r, np.float32)}
    pairs = [("rank", [2, 3]), ("reg_param", [0.05])]
    got = O.cross_validate(ratings, pairs, num_folds=3, metric=metric, cold_start_strategy=strategy, seed=4,
                           max_iter=2, als_seed=7)
    fm = []
    for tr, va in collab.k_fold(len(u), 3, 4):
        row = []
        for rank in (2, 3):
            uids, uf, mids, mf = X.fit(u[tr], m[tr], ratings["rating"][tr], rank=rank, max_iter=2, reg_param=0.05,
                                       seed=7)
            model = collab.AlsModel(uids, uf, mids, mf)
            rows, pred = model.transform({"userId": u[va], "movieId": m[va]}, strategy)
            row.append(collab.METRICS[metric](ratings["rating"][va][rows], pred))
        fm.append(row)
    assert repr(got["fold_metrics"]) == repr(fm)
    assert repr(got["avg_metrics"]) == repr(collab.average_metrics(fm))
    assert got["best_index"] == collab.best_index(got["avg_metrics"])
    assert got["param_maps"] == [dict(rank=2, max_iter=2, reg_param=0.05), dict(rank=3, max_iter=2, reg_param=0.05)]


# ---- the ABI's device-free rejections ---------------------------------------------------------------------------
def _raw_folds(u, m, r, fold, n_folds, models, cap=64):
    lib = _lib.load()
    u, m = np.ascontiguousarray(u, np.int32), np.ascontiguousarray(m, np.int32)
    r, fold = np.ascontiguousarray(r, np.float32), np.ascontiguousarray(fold, np.int32)
    M = len(models)
    specs = (_lib.SrsAlsModel * max(M, 1))(*[_lib.SrsAlsModel(*p) for p in models])
    ui, mi = np.zeros(cap * 65, np.int32), np.zeros(cap * 65, np.int32)
    uf, mf = np.zeros(cap * 64 * 65, np.float32), np.zeros(cap * 64 * 65, np.float32)
    nu, nm = np.full(65, -1, np.int32), np.full(65, -1, np.int32)
    rc = lib.srs_als_fit_folds_host(u.ctypes.data, m.ctypes.data, r.ctypes.data, fold.ctypes.data, len(u), n_folds,
                                    specs, M, 0, 0, cap, cap, ui.ctypes.data, uf.ctypes.data, nu.ctypes.data,
                                    mi.ctypes.data, mf.ctypes.data, nm.ctypes.data)
    return rc, lib.srs_last_error().decode()


def test_batched_fit_rejects_bad_inputs_before_any_device_call():
    u, m, r, fold = [1, 2, 3], [3, 4, 3], [4.0, 5.0, 3.0], [0, 1, 1]
    ok = (10, 5, 0.01, 0)
    INV = _lib.SRS_ERR_INVALID
    n0 = launch_count()
    cases = {
        "n_folds": (fold, 1, [ok]),                                          # k < 2
        "n_models 0": (fold, 2, []),                                         # an empty grid
        "n_models 65": (fold, 2, [ok] * 65),
        "rank 0": (fold, 2, [ok, (0, 5, 0.01, 0)]),
        "rank 65": (fold, 2, [(65, 5, 0.01, 0)]),
        "reg_param -0.1": (fold, 2, [(10, 5, -0.1, 0)]),
        "reg_param nan": (fold, 2, [(10, 5, NAN, 0)]),
        "max_iter 0": (fold, 2, [(10, 0, 0.01, 0)]),
        "exclude_fold 2": (fold, 2, [(10, 5, 0.01, 2)]),
        "exclude_fold -2": (fold, 2, [(10, 5, 0.01, -2)]),
        "fold 2": ([0, 2, 1], 2, [ok]),                                      # a fold id out of range
        "fold -1": ([0, -1, 1], 2, [ok]),
        "no training ratings": ([1, 1, 1], 2, [ok, (10, 5, 0.01, 1)]),      # an empty training set
    }
    for want, (f, k, models) in cases.items():
        rc, msg = _raw_folds(u, m, r, f, k, models)
        assert rc == INV and want in msg, (want, msg)
    assert _raw_folds([1, -2, 3], m, r, fold, 2, [ok])[0] == INV
    assert _raw_folds(u, m, [4.0, NAN, 1.0], fold, 2, [ok])[0] == INV
    assert _raw_folds([], [], [], [], 2, [ok])[0] == INV
    assert "model 1" in _raw_folds(u, m, r, fold, 2, [ok, (0, 5, 0.01, 0)])[1]
    assert launch_count() == n0
