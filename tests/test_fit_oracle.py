"""CPU checks of NeuralCF `fit`'s oracle (oracle/ncf_train.py), its fixtures and the trainer ABI's up-front
rejections (DESIGN.md section 4.8)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import ncf_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def small_case(seed, B, hidden=(6, 5), E=3, Vm=7, Vu=9):
    spec = default_spec("neuralcf", emb_dim=E, n_movies=Vm, n_users=Vu, hidden=hidden)
    W = {k: v.astype(np.float64) for k, v in init_weights(spec, seed, for_test=True).items()}
    rng = np.random.default_rng(seed + 100)
    for k in W:                                               # larger scale, so relus switch on both sides
        W[k] = W[k] * 2.0 + (rng.normal(0, 0.3, W[k].shape) if k.endswith("bias") else 0)
    mid = rng.integers(0, Vm, B)
    uid = rng.integers(0, Vu, B)
    mid[: B // 2] = mid[0]                                    # repeated ids
    y = rng.integers(0, 2, B)
    return W, mid, uid, y


@pytest.mark.parametrize("seed,B", [(0, 1), (1, 5), (2, 12), (3, 33)])
def test_backward_matches_central_differences(seed, B):
    W, mid, uid, y = small_case(seed, B)
    g, _, _ = ncf_train.gradients(W, mid, uid, y, np.float64)
    h = 1e-6
    for name, w in W.items():
        num = np.zeros_like(w)
        for i in np.ndindex(w.shape):
            old = w[i]
            w[i] = old + h
            lp = ncf_train.batch_loss(W, mid, uid, y)
            w[i] = old - h
            lm = ncf_train.batch_loss(W, mid, uid, y)
            w[i] = old
            num[i] = (lp - lm) / (2 * h)
        np.testing.assert_allclose(g[name], num, rtol=1e-5, atol=1e-8, err_msg=name)


def test_partial_last_batch_divides_by_its_own_size():
    W, mid, uid, y = small_case(4, 12)
    order = np.arange(12)[None, :]
    # 12 rows at batch 5: steps of 5, 5 and 2 rows; the third step's gradient is the mean over its 2 rows
    W5, _, out, _ = ncf_train.fit(W, mid, uid, y, order, 5, np.float64, max_steps=2, keep_outputs=True)
    g, _, _ = ncf_train.gradients(W5, mid[10:], uid[10:], y[10:], np.float64)
    g2 = [ncf_train.gradients(W5, mid[i:i + 1], uid[i:i + 1], y[i:i + 1], np.float64)[0] for i in (10, 11)]
    for k in g:
        np.testing.assert_allclose(g[k], (g2[0][k] + g2[1][k]) / 2, rtol=1e-12, atol=1e-15)


def test_adam_first_step_moves_each_parameter_by_lr_sign_g():
    W, mid, uid, y = small_case(5, 12)
    g, _, _ = ncf_train.gradients(W, mid, uid, y, np.float64)
    W1 = {k: v.copy() for k, v in W.items()}
    ncf_train.Adam(W1, np.float64).step(W1, g)
    for k in W:
        d = W1[k] - W[k]
        # t = 1: m = 0.1 g, v = 0.001 g^2, alpha = lr sqrt(0.001) / 0.1, so the step is
        # lr g / (|g| + epsilon / sqrt(0.001)): lr sign(g) once |g| >> 3.2e-6
        np.testing.assert_allclose(d, -0.001 * g[k] / (np.abs(g[k]) + 1e-7 / np.sqrt(0.001)), rtol=1e-9,
                                   atol=1e-18, err_msg=k)
        big = np.abs(g[k]) > 1e-3
        assert big.any(), k
        np.testing.assert_allclose(d[big], -0.001 * np.sign(g[k][big]), rtol=4e-3, err_msg=k)
        assert np.all(d[g[k] == 0] == 0), k


def test_table_row_absent_from_step_two_still_moves():
    """Keras's sparse Adam decays m and v of every row and updates every row: a movie row of the step-1 batch that
    step 2 does not contain still moves at step 2 (by about lr * beta_1 m / sqrt(beta_2 v)).  Lazy Adam leaves it."""
    W, mid, uid, y = small_case(6, 4)
    mid = np.array([1, 1, 2, 3]); uid = np.array([0, 1, 2, 3])
    orders = np.array([[0, 1, 2, 3]])
    # step 1: rows 0, 1 (movie 1); step 2: rows 2, 3 (movies 2 and 3)
    moved = {}
    for lazy in (False, True):
        W1, _, _, _ = ncf_train.fit(W, mid, uid, y, orders, 2, np.float64, lazy=lazy, max_steps=1)
        W2, _, _, _ = ncf_train.fit(W, mid, uid, y, orders, 2, np.float64, lazy=lazy, max_steps=2)
        moved[lazy] = W2["movieId_embedding"][1] - W1["movieId_embedding"][1]
    t = 2
    alpha = 0.001 * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
    g1, _, _ = ncf_train.gradients(W, mid[:2], uid[:2], y[:2], np.float64)
    G = g1["movieId_embedding"][1]
    expect = -alpha * (0.9 * 0.1 * G) / (np.sqrt(0.999 * 0.001 * G * G) + 1e-7)
    np.testing.assert_allclose(moved[False], expect, rtol=1e-9)
    assert np.all(np.abs(moved[False]) > 1e-4)
    assert np.all(moved[True] == 0)


def test_float32_oracle_tracks_float64():
    W, mid, uid, y = small_case(7, 40)
    orders = ncf_train.epoch_orders(40, 2, 7)
    W64, h64, _, _ = ncf_train.fit(W, mid, uid, y, orders, 12, np.float64)
    W32, h32, _, _ = ncf_train.fit(W, mid, uid, y, orders, 12, np.float32)
    for k in W:
        assert np.abs(W32[k] - W64[k]).max() < 1e-5, k
    assert abs(h32[-1]["loss"] - h64[-1]["loss"]) < 1e-5


def test_epoch_orders_match_the_trainer():
    from sparrowrecsys_b200.training import epoch_orders
    assert np.array_equal(epoch_orders(1000, 3, 5), ncf_train.epoch_orders(1000, 3, 5))
    assert all(np.array_equal(np.sort(o), np.arange(1000)) for o in epoch_orders(1000, 3, 5))


def test_train_fixtures():
    z = np.load(os.path.join(GOLDEN, "neuralcf_trainset.npz"))
    assert z["label"].shape == (88827,) and set(np.unique(z["label"])) == {0, 1}
    assert z["movieId"].max() < 1001 and z["userId"].max() < 30001 and z["movieId"].min() >= 0
    with open(os.path.join(GOLDEN, "neuralcf_fit.json")) as f:
        fit = json.load(f)
    assert fit["rows"] == 88827 and fit["epochs"] == 5 and fit["batch_size"] == 12
    assert [r["seed"] for r in fit["runs"]] == fit["seeds"] and 0 in fit["seeds"]
    for r in fit["runs"]:
        assert r["iterations"] == 5 * 7403 and len(r["history"]) == 5
        for k, (lo, hi) in fit["band"].items():
            assert lo <= r["test"][k] <= hi


@pytest.mark.skipif(not os.path.exists("/root/reference/src/main/resources/webroot/sampledata/trainingSamples.csv"),
                    reason="needs the reference checkout")
def test_generator_reproduces_trainset():
    import subprocess
    import sys
    subprocess.check_call([sys.executable, os.path.join(GOLDEN, "make_train_golden.py"), "--check"])


# ---- the trainer ABI's rejections that need no device ----------------------------------------------------------
def _lib_or_skip():
    from sparrowrecsys_b200 import _lib
    try:
        return _lib, _lib.load()
    except ImportError as e:
        pytest.skip(str(e))


def test_trainer_rejects_other_models_before_any_device_call():
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    for model in ("twotowers", "din", "embeddingmlp"):
        sp = _spec_struct(default_spec(model))
        out = C.c_void_p()
        rc = lib.srs_trainer_create(C.byref(sp), None, 0, 0, None, C.byref(out))
        assert rc == _lib.SRS_ERR_INVALID and not out.value
        assert b"NeuralCF" in lib.srs_last_error()


@pytest.mark.parametrize("hp", [dict(lr=0.0), dict(beta_1=1.0), dict(beta_2=-0.1), dict(epsilon=0.0)])
def test_trainer_rejects_bad_adam_hyperparameters(hp):
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    sp = _spec_struct(default_spec("neuralcf"))
    a = _lib.SrsAdam(**dict(ncf_train.KERAS_ADAM, **hp))
    out = C.c_void_p()
    assert lib.srs_trainer_create(C.byref(sp), None, 0, 0, C.byref(a), C.byref(out)) == _lib.SRS_ERR_INVALID


def test_trainer_rejects_unsupported_widths():
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    for spec in (default_spec("neuralcf", hidden=(40, 10)), default_spec("neuralcf", hidden=(10, 10, 10, 10))):
        sp = _spec_struct(spec)
        out = C.c_void_p()
        assert lib.srs_trainer_create(C.byref(sp), None, 0, 0, None, C.byref(out)) == _lib.SRS_ERR_INVALID
