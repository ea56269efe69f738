"""CPU checks of DeepFM `fit`'s oracle (oracle/deepfm_train.py), its fixtures and the trainer ABI's up-front
rejections for DeepFM (DESIGN.md section 4.9)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import ctr_oracle, deepfm_train, ncf_train
from sparrowrecsys_b200.spec import NUMERIC_KEYS, default_spec
from sparrowrecsys_b200.weights import init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def small_case(seed, B, hidden=(6, 5), E=3, Vm=7, Vu=9):
    """A small DeepFM with repeated ids and missing genres, at scales where the relus switch on both sides."""
    spec = default_spec("deepfm", emb_dim=E, n_movies=Vm, n_users=Vu, hidden=hidden)
    G = spec.n_genres
    W = {k: v.astype(np.float64) for k, v in init_weights(spec, seed, for_test=True).items()}
    rng = np.random.default_rng(seed + 100)
    for k in W:
        W[k] = W[k] * 2.0 + (rng.normal(0, 0.3, W[k].shape) if k.endswith("bias") else 0)
    mid = rng.integers(0, Vm, B)
    uid = rng.integers(0, Vu, B)
    ig = rng.integers(-1, G, B)
    ug = rng.integers(-1, G, B)
    mid[: B // 2] = mid[0]                                    # repeated ids
    ig[: B // 3] = ig[0]
    ug[-1] = -1                                               # a missing userGenre1
    num = rng.normal(0, 1, (B, 7)).astype(np.float32)
    y = rng.integers(0, 2, B)
    return spec, W, deepfm_train.Rows(mid, uid, ig, ug, num), y


def _features(r):
    f = {"movieId": r.mid, "userId": r.uid, "movieGenre1": r.ig, "userGenre1": r.ug}
    f.update({k: r.num[:, j] for j, k in enumerate(NUMERIC_KEYS)})
    return f


@pytest.mark.parametrize("seed,B", [(0, 12), (1, 33)])
def test_forward_is_ctr_oracle_deepfm_forward(seed, B):
    spec, W, r, _ = small_case(seed, B)
    p, z, _ = deepfm_train.forward(W, r, np.float64)
    po, zo = ctr_oracle.deepfm_forward(spec, W, _features(r), np.float64)
    np.testing.assert_allclose(z, zo[:, 0], rtol=0, atol=1e-12)
    np.testing.assert_allclose(p, po[:, 0], rtol=0, atol=1e-12)


def test_forward_on_the_testset_is_ctr_oracle_deepfm_forward():
    z = dict(np.load(os.path.join(GOLDEN, "dien_testset.npz")))
    spec = default_spec("deepfm")
    W = init_weights(spec, 1, for_test=False)
    f = {k: v[:2000] for k, v in z.items()}
    assert (f["userGenre1"] < 0).any()
    _, zz, _ = deepfm_train.forward(W, deepfm_train.Rows.from_features(f), np.float64)
    _, zo = ctr_oracle.deepfm_forward(spec, W, f, np.float64)
    np.testing.assert_allclose(zz, zo[:, 0], rtol=0, atol=1e-12)


@pytest.mark.parametrize("seed,B", [(0, 1), (1, 5), (2, 12)])
def test_backward_matches_central_differences(seed, B):
    _, W, r, y = small_case(seed, B)
    g, _, _ = deepfm_train.gradients(W, r, y, np.float64)
    h = 1e-6
    for name, w in W.items():
        num = np.zeros_like(w)
        for i in np.ndindex(w.shape):
            old = w[i]
            w[i] = old + h
            lp = deepfm_train.batch_loss(W, r, y)
            w[i] = old - h
            lm = deepfm_train.batch_loss(W, r, y)
            w[i] = old
            num[i] = (lp - lm) / (2 * h)
        np.testing.assert_allclose(g[name], num, rtol=1e-5, atol=1e-8, err_msg=name)


def test_missing_genre_gives_no_gradient():
    _, W, r, y = small_case(3, 6)
    r.ig[:] = -1
    r.ug[:] = -1
    g, _, _ = deepfm_train.gradients(W, r, y, np.float64)
    assert not g["fm_movieGenre1_embedding"].any() and not g["fm_userGenre1_embedding"].any()
    G = W["fm_movieGenre1_embedding"].shape[0]
    Vm = W["fm_movieId_embedding"].shape[0]
    K = g["dense_2/kernel"][:, 0]
    assert not K[:G].any() and not K[G + Vm:2 * G + Vm].any()      # the genre one-hot rows
    assert K[G:G + Vm].any()


def test_partial_last_batch_divides_by_its_own_size():
    _, W, r, y = small_case(4, 12)
    order = np.arange(12)[None, :]
    W5, _, _, _ = deepfm_train.fit(W, r, y, order, 5, np.float64, max_steps=2)
    g, _, _ = deepfm_train.gradients(W5, r.take(np.arange(10, 12)), y[10:], np.float64)
    g2 = [deepfm_train.gradients(W5, r.take(np.array([i])), y[i:i + 1], np.float64)[0] for i in (10, 11)]
    for k in g:
        np.testing.assert_allclose(g[k], (g2[0][k] + g2[1][k]) / 2, rtol=1e-12, atol=1e-15, err_msg=k)


def test_adam_first_step_moves_each_parameter_by_lr_sign_g():
    _, W, r, y = small_case(5, 12)
    g, _, _ = deepfm_train.gradients(W, r, y, np.float64)
    W1 = {k: v.copy() for k, v in W.items()}
    deepfm_train.Adam(W1, np.float64).step(W1, g)
    for k in W:
        d = W1[k] - W[k]
        np.testing.assert_allclose(d, -0.001 * g[k] / (np.abs(g[k]) + 1e-7 / np.sqrt(0.001)), rtol=1e-9,
                                   atol=1e-18, err_msg=k)
        assert np.all(d[g[k] == 0] == 0), k


def _two_steps(W, r, y, lazy):
    orders = np.array([np.arange(len(y))])
    W1, _, _, _ = deepfm_train.fit(W, r, y, orders, 2, np.float64, lazy=lazy, max_steps=1)
    W2, _, _, _ = deepfm_train.fit(W, r, y, orders, 2, np.float64, lazy=lazy, max_steps=2)
    return W1, W2


def _moved_by_decay(G):
    """What a parameter with step-1 gradient G and no step-2 gradient moves by at step 2 (m = 0.09 G,
    v = 0.000999 G^2 under either form)."""
    alpha = 0.001 * np.sqrt(1 - 0.999 ** 2) / (1 - 0.9 ** 2)
    return -alpha * (0.9 * 0.1 * G) / (np.sqrt(0.999 * 0.001 * G * G) + 1e-7)


def test_one_hot_row_absent_from_step_two_moves_by_the_dense_form():
    """dense_2/kernel is a dense variable (the indicator column's gradient is a MatMul gradient): a one-hot row of
    the step-1 batch that step 2 does not select still moves at step 2, lazy or not."""
    _, W, r, y = small_case(6, 4)
    r.mid[:] = [1, 1, 2, 3]
    G_ = W["fm_movieGenre1_embedding"].shape[0]
    g1, _, _ = deepfm_train.gradients(W, r.take(np.arange(2)), y[:2], np.float64)
    row = G_ + 1                                              # movieId 1's one-hot row
    expect = _moved_by_decay(g1["dense_2/kernel"][row, 0])
    for lazy in (False, True):
        W1, W2 = _two_steps(W, r, y, lazy)
        moved = W2["dense_2/kernel"][row, 0] - W1["dense_2/kernel"][row, 0]
        np.testing.assert_allclose(moved, expect, rtol=1e-9)
        assert abs(moved) > 1e-4
    # the dense form itself: m += (g - m)(1 - b1) with g = 0
    opt = deepfm_train.Adam({"k": np.zeros(1)}, np.float64)
    opt.m["k"][0], opt.v["k"][0] = 0.3, 0.02
    w = {"k": np.zeros(1)}
    opt.iterations = 1
    opt.step(w, {"k": np.zeros(1)})
    assert opt.m["k"][0] == 0.3 + (0 - 0.3) * (1 - 0.9) and opt.v["k"][0] == 0.02 + (0 - 0.02) * (1 - 0.999)


def test_table_row_absent_from_step_two_moves_by_the_sparse_form():
    _, W, r, y = small_case(7, 4)
    r.mid[:] = [1, 1, 2, 3]
    g1, _, _ = deepfm_train.gradients(W, r.take(np.arange(2)), y[:2], np.float64)
    moved = {}
    for lazy in (False, True):
        W1, W2 = _two_steps(W, r, y, lazy)
        moved[lazy] = {k: W2[k][1] - W1[k][1] for k in ("fm_movieId_embedding", "deep_movieId_embedding")}
    for k in ("fm_movieId_embedding", "deep_movieId_embedding"):
        np.testing.assert_allclose(moved[False][k], _moved_by_decay(g1[k][1]), rtol=1e-9, err_msg=k)
        assert np.all(np.abs(moved[False][k]) > 1e-4), k
        assert np.all(moved[True][k] == 0), k
    # the sparse form itself: m = b1 m + (1 - b1) g on a table
    opt = deepfm_train.Adam({"fm_movieId_embedding": np.zeros(1)}, np.float64)
    opt.m["fm_movieId_embedding"][0] = 0.3
    opt.step({"fm_movieId_embedding": np.zeros(1)}, {"fm_movieId_embedding": np.zeros(1)})
    assert opt.m["fm_movieId_embedding"][0] == 0.9 * 0.3 + (1 - 0.9) * 0


def test_adam_matches_ncf_train_adam_off_the_tables():
    """DeepFM's Adam is NeuralCF's on every tensor that is not a table: the same state, alpha and dense form."""
    rng = np.random.default_rng(3)
    W = {"dense/kernel": rng.normal(size=(4, 3)), "userId_embedding": rng.normal(size=(5, 2))}
    g = {k: rng.normal(size=v.shape) for k, v in W.items()}
    g["userId_embedding"][1] = 0
    for dt in (np.float32, np.float64):
        a, b = ({k: v.astype(dt) for k, v in W.items()} for _ in range(2))
        oa, ob = deepfm_train.Adam(a, dt), ncf_train.Adam(b, dt)
        for _ in range(3):
            oa.step(a, g)
            ob.step(b, g)
        assert np.array_equal(a["dense/kernel"], b["dense/kernel"])
        assert np.array_equal(oa.v["dense/kernel"], ob.v["dense/kernel"]) and oa.iterations == ob.iterations == 3
        # userId_embedding is a NeuralCF table but a dense DeepFM name: the two forms part ways only in the last bits
        np.testing.assert_allclose(a["userId_embedding"], b["userId_embedding"], rtol=1e-5)


def test_float32_oracle_tracks_float64():
    _, W, r, y = small_case(8, 40)
    orders = deepfm_train.epoch_orders(40, 2, 7)
    W64, h64, _, _ = deepfm_train.fit(W, r, y, orders, 12, np.float64)
    W32, h32, _, _ = deepfm_train.fit(W, r, y, orders, 12, np.float32)
    for k in W:
        assert np.abs(W32[k] - W64[k]).max() < 1e-5, k
    assert abs(h32[-1]["loss"] - h64[-1]["loss"]) < 1e-5


def test_train_fixtures():
    z = np.load(os.path.join(GOLDEN, "deepfm_trainset.npz"))
    assert sorted(z.files) == sorted(["movieId", "userId", "label", *NUMERIC_KEYS, "movieGenre1", "userGenre1"])
    assert z["label"].shape == (88827,) and set(np.unique(z["label"])) == {0, 1}
    assert z["movieGenre1"].dtype == np.int8 and z["userGenre1"].dtype == np.int8
    assert z["movieId"].max() < 1001 and z["userId"].max() < 30001 and z["movieId"].min() >= 0
    assert z["movieGenre1"].max() < 19 and z["userGenre1"].max() < 19
    assert (z["userGenre1"] < 0).sum() == 1227
    n = np.load(os.path.join(GOLDEN, "neuralcf_trainset.npz"))  # the same rows in the same order
    assert all(np.array_equal(z[k], n[k]) for k in ("movieId", "userId", "label"))
    with open(os.path.join(GOLDEN, "deepfm_fit.json")) as f:
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
    subprocess.check_call([sys.executable, os.path.join(GOLDEN, "make_deepfm_train_golden.py"), "--check"])


# ---- the trainer ABI's rejections that need no device ----------------------------------------------------------
def _lib_or_skip():
    from sparrowrecsys_b200 import _lib
    try:
        return _lib, _lib.load()
    except ImportError as e:
        pytest.skip(str(e))


def _create(spec, hp=None, **fields):
    """srs_trainer_create with no tensors; `fields` override the srs_spec struct (shapes ModelSpec refuses)."""
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    sp = _spec_struct(spec)
    for k, v in fields.items():
        setattr(sp, k, v)
    out = C.c_void_p()
    rc = lib.srs_trainer_create(C.byref(sp), None, 0, 0, None if hp is None else C.byref(hp), C.byref(out))
    assert not out.value
    return _lib, lib, rc


@pytest.mark.parametrize("overrides", [dict(hidden=(64,)), dict(hidden=(64, 64, 64)), dict(hidden=(65, 64)),
                                       dict(hidden=(64, 65)), dict(hidden=(0, 64))])
def test_trainer_rejects_unsupported_deepfm_shapes(overrides):
    _lib, lib, rc = _create(default_spec("deepfm", **overrides))
    assert rc == _lib.SRS_ERR_INVALID


def test_trainer_rejects_deepfm_emb_dim_65():
    _lib, lib, rc = _create(default_spec("deepfm", emb_dim=64), emb_dim=65)
    assert rc == _lib.SRS_ERR_INVALID and b"emb_dim" in lib.srs_last_error()


@pytest.mark.parametrize("hp", [dict(lr=0.0), dict(beta_1=1.0), dict(beta_2=-0.1), dict(epsilon=0.0)])
def test_trainer_rejects_bad_adam_hyperparameters_for_deepfm(hp):
    _lib, _ = _lib_or_skip()
    a = _lib.SrsAdam(**dict(ncf_train.KERAS_ADAM, **hp))
    _lib, lib, rc = _create(default_spec("deepfm"), a)
    assert rc == _lib.SRS_ERR_INVALID


def test_trainer_still_rejects_other_models_naming_neuralcf():
    for model in ("deepfm_v2", "widendeep", "dien"):
        _lib, lib, rc = _create(default_spec(model))
        assert rc == _lib.SRS_ERR_INVALID
        assert b"NeuralCF" in lib.srs_last_error() and b"DeepFM" in lib.srs_last_error()


def test_python_trainer_accepts_deepfm_and_rejects_others():
    from sparrowrecsys_b200.training import Trainer
    assert "deepfm" in Trainer.MODELS
    with pytest.raises(NotImplementedError, match="NeuralCF"):
        Trainer(default_spec("din"), {})
