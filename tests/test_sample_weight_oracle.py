"""Keras's `sample_weight` / `class_weight` in the weighted oracle (tests/weighted_oracle.py) and the host helper
(DESIGN.md section 4.28), without a device: the weighted backward over each training oracle against central
differences of sum w_i l_i / B; the weighted metrics against duplicated rows; the float64-parity tolerance of two
existing fit cases against the weighting mistakes a kernel could make; and `training.sample_weights`' checks."""
import numpy as np
import pytest

import weighted_oracle as WO
from oracle import deepfm_train, keras_eval
from sparrowrecsys_b200.training import sample_weights
from test_fit_matrix import DEFECT_MULTIPLE, FIT_MATRIX, FitCase, _inputs, _rows, _unit_numerics
from test_fit_oracle_twotowers import TTCase
from test_fit_oracle_twotowers import inputs as tt_inputs

ORACLE = WO.ORACLE
TINY = dict(n_movies=4, n_users=5)      # every id repeats in the batch


def row_weights(n, seed, spread=(0.2, 3.0)):
    """Weights with zeros, 0.37 and 1e3 among uniform ones, none of them 1."""
    rng = np.random.default_rng(seed)
    w = rng.uniform(*spread, n).astype(np.float32)
    w[::9] = 0.0
    w[4::17] = 0.37
    w[7 % max(n, 1)] = 1e3
    return w


# ---- the oracles' weighted backward ------------------------------------------------------------------------
def _small(model, seed, B):
    """(W float64 scaled so relus switch both ways, call(W) -> (args before dtype), labels) of a small batch."""
    if model == "twotowers":
        c = TTCase(dict(emb_dim=3, hidden=(4, 3), **TINY), B, B, 1, seed, None)
        W0, f, _ = tt_inputs(c)
        args = (f["movieId"], f["userId"])
    else:
        hidden = {"neuralcf": (4, 3), "deepfm": (5, 4), "widendeep": (5, 4), "deepfm_v2": (5, 4)}[model]
        c = FitCase(model, dict(emb_dim=3, hidden=hidden, **TINY), B, B, 1, seed, None)
        W0, f = _inputs(c)[:2]
        if model == "deepfm":          # the golden rows' raw numerics put relu kinks within a difference step
            f = dict(f, **_unit_numerics(np.random.default_rng(seed), B))
            args = (deepfm_train.Rows.from_features(f),)
        else:
            args = (f["movieId"], f["userId"]) if model == "neuralcf" else (_rows(c),)
    rng = np.random.default_rng(seed + 100)
    W = {k: v.astype(np.float64) * 2.0 + (rng.normal(0, 0.3, v.shape) if k.endswith("bias") else 0)
         for k, v in W0.items()}
    return W, args, np.asarray(f["label"])


def _weighted_loss(mod, W, args, y, w):
    z = mod.forward(W, *args, np.float64)[1]
    yv = y.astype(np.float64)
    return float(np.sum(w * (np.maximum(z, 0) - z * yv + np.log1p(np.exp(-np.abs(z))))) / len(y))


@pytest.mark.parametrize("model", sorted(ORACLE))
@pytest.mark.parametrize("seed,B", [(0, 45), (1, 50)])
def test_weighted_backward_matches_central_differences(model, seed, B):
    """Repeated ids (vocabularies of 4 and 5), missing genres (the rows of test_fit_matrix), weights of 0, 0.37 and
    1e3, and class_weight x sample_weight, on 24 entries of every tensor (every entry of the small ones)."""
    mod = ORACLE[model]
    W, args, y = _small(model, seed, B)
    w = sample_weights(y, row_weights(B, seed), {0: 0.5, 1: 2.0}).astype(np.float64)
    assert (w == 0).any() and (w > 100).any()
    g = WO.gradients(model, W, *args, y, np.float64, weight=w)[0]
    assert g.keys() == W.keys()
    rng = np.random.default_rng(seed)
    h = 1e-6
    for name, t in W.items():
        flat = t.reshape(-1)
        picks = np.arange(flat.size) if flat.size <= 24 else rng.choice(flat.size, 24, replace=False)
        gf = g[name].reshape(-1)
        for i in picks:
            old = flat[i]
            flat[i] = old + h
            lp = _weighted_loss(mod, W, args, y, w)
            flat[i] = old - h
            lm = _weighted_loss(mod, W, args, y, w)
            flat[i] = old
            num = (lp - lm) / (2 * h)
            assert abs(gf[i] - num) <= 1e-5 * abs(num) + 2e-6, (name, int(i), gf[i], num)


@pytest.mark.parametrize("model", sorted(ORACLE))
def test_unit_weights_give_the_unweighted_gradients_bit_for_bit(model):
    W, args, y = _small(model, 2, 41)
    for dtype in (np.float32, np.float64):
        g0 = ORACLE[model].gradients(W, *args, y, dtype)[0]
        g1 = WO.gradients(model, W, *args, y, dtype, weight=np.ones(len(y), np.float32))[0]
        for k in g0:
            assert np.array_equal(g0[k], g1[k]), (model, k)


def test_zero_weight_rows_add_no_gradient():
    W, args, y = _small("deepfm", 3, 45)
    w = np.ones(45)
    w[10:] = 0.0
    gw = WO.gradients("deepfm", W, *args, y, np.float64, weight=w)[0]
    # the first 10 rows alone, still divided by all 45
    head = deepfm_train.gradients(W, args[0].take(np.arange(10)), y[:10], np.float64)[0]
    for k in gw:
        np.testing.assert_allclose(gw[k], head[k] * 10 / 45, rtol=1e-12, atol=1e-15, err_msg=k)


# ---- keras_eval's weighted metrics -------------------------------------------------------------------------
def _scores(n, seed):
    rng = np.random.default_rng(seed)
    p = rng.random(n).astype(np.float32)
    p[:8] = keras_eval.keras_thresholds()[[0, 1, 50, 99, 100, 150, 198, 199]].clip(0, 1)   # on the thresholds
    p[8] = 0.5
    z = np.log(np.maximum(p, 1e-6) / np.maximum(1 - p, 1e-6)).astype(np.float32)
    y = (rng.random(n) < 0.4).astype(np.int32)
    return p, z, y


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_integer_weights_are_duplicated_rows(seed):
    p, z, y = _scores(3000, seed)
    w = np.random.default_rng(seed + 9).integers(0, 5, 3000).astype(np.float32)
    rw = WO.keras_evaluate(p, z, y, w)
    k = w.astype(np.int64)
    rd = WO.keras_evaluate(np.repeat(p, k), np.repeat(z, k), np.repeat(y, k))
    for key in ("accuracy", "roc_auc", "pr_auc"):
        assert rw[key] == rd[key], key
    for key in ("tp", "fp", "tn", "fn"):
        assert np.array_equal(rw[key], rd[key].astype(np.float64)), key
    assert (rw["rows"], rw["positives"], rw["correct"]) == (3000, int(y.sum()), int((y == (p > 0.5)).sum()))


def test_weighted_loss_is_over_the_row_count():
    p, z, y = _scores(500, 4)
    w = row_weights(500, 4)
    r = WO.keras_evaluate(p, z, y, w)
    l32 = keras_eval.logit_bce_f32(z, y)
    assert r["loss"] == float(np.sum((w * l32).astype(np.float64)) / 500)
    assert r["loss"] != float(np.sum((w * l32).astype(np.float64)) / np.sum(w.astype(np.float64)))


def test_all_ones_weights_are_the_unweighted_metrics_bit_for_bit():
    p, z, y = _scores(2000, 5)
    r0 = WO.keras_evaluate(p, z, y)
    r1 = WO.keras_evaluate(p, z, y, np.ones(2000, np.float32))
    for key in ("loss", "accuracy", "roc_auc", "pr_auc", "rows", "positives", "correct"):
        assert r0[key] == r1[key], key


def test_zero_weights_give_zero_accuracy():
    p, z, y = _scores(50, 6)
    r = WO.keras_evaluate(p, z, y, np.zeros(50, np.float32))
    assert (r["loss"], r["accuracy"], r["roc_auc"], r["pr_auc"]) == (0.0, 0.0, 0.0, 0.0)


# ---- the parity tolerance sees weighting mistakes ----------------------------------------------------------
DEFECT_CASES = [FIT_MATRIX[0], FIT_MATRIX[13]]      # NeuralCF <12, 16> and DeepFM EP 16 at B 33


def _weighted_fit(c, dtype, w):
    W0, f, orders = _inputs(c)
    data = (f["movieId"], f["userId"]) if c.model == "neuralcf" else _rows(c)
    return WO.fit(c.model, W0, data, f["label"], orders, c.B, dtype, hp=c.adam, weights=w)[0]


@pytest.mark.parametrize("case", DEFECT_CASES, ids=lambda c: "%s-B%d-n%d" % (c.model, c.B, c.n))
def test_tolerance_sees_each_weighting_mistake(case, monkeypatch):
    """The GPU test's rule (the case's multiple of the float32 oracle's distance from float64, plus one ulp) on the
    weighted fit: a weight dropped on one row of each batch, a weight applied twice and a division by sum w instead
    of B each move some tensor by more than DEFECT_MULTIPLE tolerances."""
    w = row_weights(case.n, case.seed)
    W64, W32 = _weighted_fit(case, np.float64, w), _weighted_fit(case, np.float32, w)
    tol = {k: case.multiple * float(np.abs(W32[k] - W64[k]).max())
           + float(np.spacing(np.float32(np.abs(W64[k]).max()))) for k in W64}
    intact = WO.numerator

    def dropped(p, y, w, dtype):                 # the last row of each batch unweighted
        w = np.array(w)
        w[-1] = 1.0
        return intact(p, y, w, dtype)

    def twice(p, y, w, dtype):
        return intact(p, y, np.asarray(w, np.float64) ** 2, dtype)

    def over_sum(p, y, w, dtype):                # dz = w (p - y) / sum w
        return (intact(p, y, w, dtype) * (len(w) / np.sum(np.asarray(w, np.float64)))).astype(dtype)

    assert w[case.B - 1] != 1.0
    for name, fn in (("dropped on one row", dropped), ("applied twice", twice), ("divided by sum w", over_sum)):
        monkeypatch.setattr(WO, "numerator", fn)
        Wd = _weighted_fit(case, np.float64, w)
        monkeypatch.setattr(WO, "numerator", intact)
        far = max(float(np.abs(Wd[k] - W64[k]).max()) / tol[k] for k in tol)
        assert far > DEFECT_MULTIPLE, (name, far)


# ---- the host helper --------------------------------------------------------------------------------------
def test_sample_weights_builds_keras_products():
    y = np.array([0, 1, 1, 0], np.int32)
    assert sample_weights(y) is None
    w = sample_weights(y, [1.0, 2.0, 0.5, 0.0], {0: 3.0, 1: 0.25})
    assert w.dtype == np.float32 and np.array_equal(w, np.float32([3.0, 0.5, 0.125, 0.0]))
    assert np.array_equal(sample_weights(y, class_weight={1: 2}), np.float32([1, 2, 2, 1]))
    assert np.array_equal(sample_weights(y, np.array([[1], [2], [3], [4]])), np.float32([1, 2, 3, 4]))


@pytest.mark.parametrize("kwargs", [
    dict(sample_weight=[1.0, 2.0, 3.0]),                     # a length other than the rows'
    dict(sample_weight=[[1.0, 2.0]] * 4),
    dict(sample_weight=[1.0, -0.5, 1.0, 1.0]),
    dict(sample_weight=[1.0, np.nan, 1.0, 1.0]),
    dict(sample_weight=[1.0, np.inf, 1.0, 1.0]),
    dict(sample_weight=[1.0, 1e39, 1.0, 1.0]),               # infinite in float32
    dict(sample_weight=["a", "b", "c", "d"]),
    dict(class_weight={2: 1.0}),
    dict(class_weight={True: 1.0}),
    dict(class_weight={"1": 1.0}),
    dict(class_weight={0: -1.0}),
    dict(class_weight={1: np.nan}),
    dict(class_weight=[1.0, 2.0]),
    dict(sample_weight=[1.0, 1e30, 1.0, 1.0], class_weight={1: 1e10}),   # a product past float32
])
def test_sample_weights_rejects(kwargs):
    with pytest.raises(ValueError):
        sample_weights(np.array([0, 1, 1, 0], np.int32), **kwargs)
