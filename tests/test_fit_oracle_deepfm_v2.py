"""CPU checks of DeepFM_v2 `fit`'s oracle (oracle/deepfm_v2_train.py), its known answers, the step kernel's dispatch
and the trainer ABI's up-front rejections for DeepFM_v2 (DESIGN.md section 4.19)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import ctr_oracle, deepfm_v2_train, keras_eval, ncf_train
from sparrowrecsys_b200.spec import MODEL_KINDS, default_spec
from sparrowrecsys_b200.weights import init_weights

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
T = deepfm_v2_train


def small_case(seed, B, hidden=(6, 5), E=3, Vm=7, Vu=9):
    """A small DeepFM_v2 with repeated ids, two rows on one movie and a missing genre in each genre field, at scales
    where the relus switch on both sides."""
    spec = default_spec("deepfm_v2", emb_dim=E, n_movies=Vm, n_users=Vu, hidden=hidden)
    G = spec.n_genres
    W = {k: v.astype(np.float64) for k, v in init_weights(spec, seed, for_test=True).items()}
    rng = np.random.default_rng(seed + 100)
    for k in W:
        W[k] = W[k] * 2.0 + (rng.normal(0, 0.3, W[k].shape) if k.endswith("bias") else 0)
    mid = rng.integers(0, Vm, B)
    uid = rng.integers(0, Vu, B)
    ig = rng.integers(0, G, B)
    ug = rng.integers(0, G, B)
    uid[: B // 2] = uid[0]                                    # repeated ids
    if B > 1:
        mid[1] = mid[0]                                       # two rows on one movie
        ig[-1] = -1                                           # a missing genre in each field
        ug[-2] = -1
    num = rng.normal(0, 1, (B, 7)).astype(np.float32)
    y = rng.integers(0, 2, B)
    return spec, W, T.Rows(mid, uid, ig, ug, num), y


@pytest.mark.parametrize("seed,B", [(0, 12), (1, 33)])
def test_forward_is_ctr_oracle_deepfm_v2_forward(seed, B):
    spec, W, r, _ = small_case(seed, B)
    p, z, _ = T.forward(W, r, np.float64)
    po, zo = ctr_oracle.deepfm_v2_forward(spec, W, T.features(r), np.float64)
    np.testing.assert_allclose(z, zo[:, 0], rtol=0, atol=1e-12)
    np.testing.assert_allclose(p, po[:, 0], rtol=0, atol=1e-12)


def _load(part):
    return dict(np.load(os.path.join(GOLDEN, "deepfm_trainset.npz" if part == "train" else "dien_testset.npz")))


def test_forward_on_the_testset_is_ctr_oracle_deepfm_v2_forward():
    """The raw numerics (rating counts up to 14 617) included: the same logits to 1e-12 relative to their size."""
    spec = default_spec("deepfm_v2")
    W = init_weights(spec, 1, for_test=False)
    f = {k: v[:2000] for k, v in _load("test").items()}
    assert (f["userGenre1"] < 0).any()
    _, z, _ = T.forward(W, T.Rows.from_features(f), np.float64)
    _, zo = ctr_oracle.deepfm_v2_forward(spec, W, f, np.float64)
    np.testing.assert_allclose(z, zo[:, 0], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("seed,B", [(0, 1), (1, 5), (2, 12)])
def test_backward_matches_central_differences(seed, B):
    _, W, r, y = small_case(seed, B)
    g, _, _ = T.gradients(W, r, y, np.float64)
    h = 1e-6
    for name, w in W.items():
        num = np.zeros_like(w)
        for i in np.ndindex(w.shape):
            old = w[i]
            w[i] = old + h
            lp = T.batch_loss(W, r, y)
            w[i] = old - h
            lm = T.batch_loss(W, r, y)
            w[i] = old
            num[i] = (lp - lm) / (2 * h)
        np.testing.assert_allclose(g[name], num, rtol=1e-5, atol=1e-8, err_msg=name)


@pytest.mark.parametrize("field", ["movieGenre1", "userGenre1"])
def test_a_missing_genre_moves_the_projection_bias_but_not_its_table_or_kernel(field):
    """A row whose genre is missing has a zero embedding column: its proj bias still gets dF, its proj kernel and
    table get nothing, and its one-hot weight gets no entry."""
    _, W, r, y = small_case(3, 1)
    setattr(r, "ig" if field == "movieGenre1" else "ug", np.array([-1]))
    g, _, _ = T.gradients(W, r, y, np.float64)
    assert not g[field + "_embedding"].any()
    assert not g["proj_%s/kernel" % field].any()
    assert np.abs(g["proj_%s/bias" % field]).max() > 1e-6
    G = W["movieGenre1_embedding"].shape[0]
    Vm = W["movieId_embedding"].shape[0]
    onehot = g["first_cat/kernel"][:, 0]
    block = slice(0, G) if field == "movieGenre1" else slice(G + Vm, 2 * G + Vm)
    assert not onehot[block].any()
    assert np.count_nonzero(onehot) == 3


def test_two_rows_on_one_movie_add_up():
    _, W, r, y = small_case(4, 2)
    r.mid[:] = 3
    g, p, _ = T.gradients(W, r, y, np.float64)
    g0, _, _ = T.gradients(W, r.take(np.array([0])), y[:1], np.float64)
    g1, _, _ = T.gradients(W, r.take(np.array([1])), y[1:], np.float64)
    np.testing.assert_allclose(g["movieId_embedding"][3], (g0["movieId_embedding"][3] + g1["movieId_embedding"][3]) / 2,
                               rtol=1e-12)
    G = W["movieGenre1_embedding"].shape[0]
    dz = (p - y) / 2
    np.testing.assert_allclose(g["first_cat/kernel"][G + 3, 0], dz.sum() * W["out/kernel"][0, 0], rtol=1e-12)


def test_partial_last_batch_divides_by_its_own_size():
    _, W, r, y = small_case(4, 12)
    order = np.arange(12)[None, :]
    W5, _, _, _ = T.fit(W, r, y, order, 5, np.float64, max_steps=2)
    g, _, _ = T.gradients(W5, r.take(np.arange(10, 12)), y[10:], np.float64)
    g2 = [T.gradients(W5, r.take(np.array([i])), y[i:i + 1], np.float64)[0] for i in (10, 11)]
    for k in g:
        np.testing.assert_allclose(g[k], (g2[0][k] + g2[1][k]) / 2, rtol=1e-12, atol=1e-15, err_msg=k)


def test_adam_first_step_moves_each_parameter_by_lr_sign_g():
    _, W, r, y = small_case(5, 12)
    g, _, _ = T.gradients(W, r, y, np.float64)
    W1 = {k: v.copy() for k, v in W.items()}
    T.Adam(W1, np.float64).step(W1, g)
    for k in W:
        d = W1[k] - W[k]
        np.testing.assert_allclose(d, -0.001 * g[k] / (np.abs(g[k]) + 1e-7 / np.sqrt(0.001)), rtol=1e-9,
                                   atol=1e-18, err_msg=k)
        assert np.all(d[g[k] == 0] == 0), k


def _two_steps(W, r, y, lazy):
    orders = np.array([np.arange(len(y))])
    W1, _, _, _ = T.fit(W, r, y, orders, 2, np.float64, lazy=lazy, max_steps=1)
    W2, _, _, _ = T.fit(W, r, y, orders, 2, np.float64, lazy=lazy, max_steps=2)
    return W1, W2


def _moved_by_decay(G):
    """What a parameter with step-1 gradient G and no step-2 gradient moves by at step 2 (m = 0.09 G,
    v = 0.000999 G^2 under either form)."""
    alpha = 0.001 * np.sqrt(1 - 0.999 ** 2) / (1 - 0.9 ** 2)
    return -alpha * (0.9 * 0.1 * G) / (np.sqrt(0.999 * 0.001 * G * G) + 1e-7)


def _absent_case(seed):
    """Four rows: step 1 (rows 0, 1) has movie 1 and movie genre 4, which step 2 (rows 2, 3) lacks."""
    spec, W, r, y = small_case(seed, 4)
    r.mid[:] = [1, 1, 2, 3]
    r.ig[:] = [4, 4, -1, 2]
    return spec, W, r, y


def test_one_hot_row_absent_from_step_two_moves_by_the_dense_form():
    """first_cat/kernel is a dense variable (the indicator columns are a dense input, so its gradient is a MatMul
    gradient): a one-hot row of the step-1 batch that step 2 does not hit still moves at step 2, lazy or not."""
    _, W, r, y = _absent_case(6)
    g1, _, _ = T.gradients(W, r.take(np.arange(2)), y[:2], np.float64)
    row = W["movieGenre1_embedding"].shape[0] + 1          # movie 1's one-hot row
    expect = _moved_by_decay(g1["first_cat/kernel"][row, 0])
    for lazy in (False, True):
        W1, W2 = _two_steps(W, r, y, lazy)
        moved = W2["first_cat/kernel"][row, 0] - W1["first_cat/kernel"][row, 0]
        np.testing.assert_allclose(moved, expect, rtol=1e-9)
        assert abs(moved) > 1e-4


def test_table_rows_absent_from_step_two_move_by_the_sparse_form_and_lazy_adam_differs():
    _, W, r, y = _absent_case(7)
    g1, _, _ = T.gradients(W, r.take(np.arange(2)), y[:2], np.float64)
    moved, final = {}, {}
    for lazy in (False, True):
        W1, W2 = _two_steps(W, r, y, lazy)
        moved[lazy] = {"movieId_embedding": W2["movieId_embedding"][1] - W1["movieId_embedding"][1],
                       "movieGenre1_embedding": W2["movieGenre1_embedding"][4] - W1["movieGenre1_embedding"][4]}
        final[lazy] = W2
    for k in moved[False]:
        row = 1 if k == "movieId_embedding" else 4
        np.testing.assert_allclose(moved[False][k], _moved_by_decay(g1[k][row]), rtol=1e-9, err_msg=k)
        assert np.all(np.abs(moved[False][k]) > 1e-4), k
        assert np.all(moved[True][k] == 0), k
    assert not np.array_equal(final[False]["movieId_embedding"], final[True]["movieId_embedding"])
    # the sparse form itself on a DeepFM_v2 table: m = b1 m + (1 - b1) g
    opt = T.Adam({"userGenre1_embedding": np.zeros(1)}, np.float64)
    opt.m["userGenre1_embedding"][0] = 0.3
    opt.step({"userGenre1_embedding": np.zeros(1)}, {"userGenre1_embedding": np.zeros(1)})
    assert opt.m["userGenre1_embedding"][0] == 0.9 * 0.3 + (1 - 0.9) * 0


def test_float32_oracle_tracks_float64():
    _, W, r, y = small_case(8, 40)
    orders = T.epoch_orders(40, 2, 7)
    W64, h64, _, _ = T.fit(W, r, y, orders, 12, np.float64)
    W32, h32, _, _ = T.fit(W, r, y, orders, 12, np.float32)
    for k in W:
        assert np.abs(W32[k] - W64[k]).max() < 1e-5, k
    assert abs(h32[-1]["loss"] - h64[-1]["loss"]) < 1e-5


def test_fit_validate_is_fit_plus_evaluate_after_the_validated_epochs():
    """deepfm_v2_train.fit_validate: the training of `fit`, bit for bit; the validated epochs' forward of the
    validation rows; epoch by epoch with the carried Adam state gives one call's bits (fit_validation.fit's rules)."""
    _, W, r, y = small_case(9, 30)
    f = dict(T.features(r), label=y)
    _, _, rv, yv = small_case(10, 20)
    val = dict(T.features(rv), label=yv)
    orders = T.epoch_orders(30, 4, 3)
    Wa, ha, va, _ = T.fit_validate(W, f, orders, 12, np.float64, val=val, validation_freq=2)
    Wb, hb, _, _ = T.fit(W, r, y, orders, 12, np.float64)
    assert ha == hb
    assert all(np.array_equal(Wa[k], Wb[k]) for k in W)
    assert va[0] is None and va[2] is None
    p, z, _ = T.forward(Wa, rv, np.float64)
    res = keras_eval.keras_evaluate(p.astype(np.float32), z.astype(np.float32), yv)
    assert va[3] == {k: res[k] for k in ("loss", "accuracy", "roc_auc", "pr_auc")}
    Wc, opt = W, None
    for e in range(4):
        Wc, _, vc, opt = T.fit_validate(Wc, f, orders[e:e + 1], 12, np.float64, val=val, opt=opt)
        if e % 2 == 1:
            assert vc[0] == va[e]
    assert all(np.array_equal(Wa[k], Wc[k]) for k in W)


# ---- what the GPU parity tolerance detects ----------------------------------------------------------------------
MULTIPLE = 4.0          # tests/test_gpu_fit_deepfm_v2.py's SPREAD_MULTIPLE


def _mutant(kind):
    """deepfm_v2_train.gradients with one deliberate mistake."""
    base = T.gradients

    def g(W, r, y, dtype=np.float32):
        if kind == "row":                                     # a dropped batch row (the last, when B > 1)
            _, p, z = base(W, r, y, dtype)
            if len(y) > 1:
                out, _, _ = base(W, r.take(np.arange(len(y) - 1)), y[:-1], dtype)
                scale = dtype((len(y) - 1) / len(y))
                return {k: v * scale for k, v in out.items()}, p, z
            return base(W, r, y, dtype)
        if kind == "fm_half":                                 # the FM with the textbook 1/2
            return base(W, r, y, dtype, fm_half=True)
        out, p, z = base(W, r, y, dtype)
        if kind == "column":                                  # a dropped embedding column
            out["userGenre1_embedding"][...] = 0
            out["proj_userGenre1/kernel"][...] = 0
        elif kind == "hidden":                                # a dropped hidden unit of the first layer
            out["deep/kernel"][:, 0] = 0
            out["deep/bias"][0] = 0
        elif kind == "onehot":                                # a dropped one-hot entry (the first row's movie)
            G = W["movieGenre1_embedding"].shape[0]
            dz = (p - np.asarray(y).astype(dtype)) / dtype(len(y))
            out["first_cat/kernel"][G + r.mid[0], 0] -= dz[0] * dtype(W["out/kernel"][0, 0])
        return out, p, z
    return g


@pytest.mark.parametrize("B,n,epochs", [(12, 115, 1), (33, 320, 1)])
def test_parity_tolerance_detects_each_mistake(monkeypatch, B, n, epochs):
    spec = default_spec("deepfm_v2")
    W0 = init_weights(spec, 3, for_test=False)                  # as the GPU parity cases of the reference shape
    f = {k: v[:n] for k, v in _load("train").items()}
    rows = T.Rows.from_features(f)
    orders = T.epoch_orders(n, epochs, 11)
    args = (W0, rows, f["label"], orders, B)
    W64, _, _, _ = T.fit(*args, dtype=np.float64)
    W32, _, _, _ = T.fit(*args, dtype=np.float32)

    def tol(k):
        return MULTIPLE * float(np.abs(W32[k] - W64[k]).max()) + float(np.spacing(np.float32(np.abs(W64[k]).max())))

    for k in W0:
        assert np.abs(W64[k] - W0[k]).max() > tol(k), k       # every tensor moves past its tolerance
    caught = {}
    for kind in ("column", "hidden", "row", "onehot", "fm_half"):
        monkeypatch.setattr(T, "gradients", _mutant(kind))
        Wm, _, _, _ = T.fit(*args, dtype=np.float64)
        monkeypatch.undo()
        caught[kind] = [k for k in W0 if np.abs(Wm[k] - W64[k]).max() > tol(k)]
    Wl, _, _, _ = T.fit(*args, dtype=np.float64, lazy=True)
    caught["lazy"] = [k for k in W0 if np.abs(Wl[k] - W64[k]).max() > tol(k)]
    for kind, names in caught.items():
        assert names, kind


def test_train_fixture():
    with open(os.path.join(GOLDEN, "deepfm_v2_fit.json")) as f:
        fit = json.load(f)
    assert fit["rows"] == 88827 and fit["test_rows"] == 22440 and fit["epochs"] == 5 and fit["batch_size"] == 12
    assert [r["seed"] for r in fit["runs"]] == fit["seeds"] and 0 in fit["seeds"]
    for r in fit["runs"]:
        assert r["iterations"] == 5 * 7403 and len(r["history"]) == 5 and r["oracle_seconds"] > 0
        for k, (lo, hi) in fit["band"].items():
            assert lo <= r["test"][k] <= hi


# ---- the trainer ABI's rejections that need no device ----------------------------------------------------------
def _lib_or_skip():
    from sparrowrecsys_b200 import _lib
    try:
        return _lib, _lib.load()
    except ImportError as e:
        pytest.skip(str(e))


def _create(spec, hp=None, **fields):
    """srs_trainer_create_any with no tensors; `fields` override the srs_spec struct (shapes ModelSpec refuses)."""
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    sp = _spec_struct(spec)
    for k, v in fields.items():
        setattr(sp, k, v)
    out = C.c_void_p()
    rc = lib.srs_trainer_create_any(C.byref(sp), None, 0, 0, None if hp is None else C.byref(hp), C.byref(out))
    assert not out.value
    return _lib, lib, rc


@pytest.mark.parametrize("overrides,fields,match", [
    (dict(hidden=(33, 16)), {}, b"1..32 and 1..16"), (dict(hidden=(32, 17)), {}, b"1..32 and 1..16"),
    (dict(hidden=(32,)), {}, b"exactly 2"), (dict(hidden=(32, 16, 8)), {}, b"exactly 2"),
    ({}, dict(proj_dim=32), b"proj_dim"), (dict(emb_dim=64), dict(emb_dim=65), b"emb_dim")])
def test_trainer_rejects_unsupported_deepfm_v2_shapes(overrides, fields, match):
    _lib, lib, rc = _create(default_spec("deepfm_v2", **overrides), **fields)
    assert rc == _lib.SRS_ERR_INVALID and match in lib.srs_last_error()


@pytest.mark.parametrize("hp", [dict(lr=0.0), dict(beta_1=1.0), dict(beta_2=-0.1), dict(epsilon=0.0)])
def test_trainer_rejects_bad_adam_hyperparameters_for_deepfm_v2(hp):
    _lib, _ = _lib_or_skip()
    a = _lib.SrsAdam(**dict(ncf_train.KERAS_ADAM, **hp))
    _lib, lib, rc = _create(default_spec("deepfm_v2"), a)
    assert rc == _lib.SRS_ERR_INVALID and b"Adam" in lib.srs_last_error()


def test_create_any_takes_exactly_the_kinds_the_python_trainer_trains():
    """The accepted list is not pinned here: for every model kind, srs_trainer_create_any rejects it up front
    (SRS_ERR_INVALID) if and only if Trainer.MODELS lacks it.  An accepted kind with no tensors fails later, on the
    device check or the first missing tensor, with another code."""
    from sparrowrecsys_b200.training import Trainer
    assert "deepfm_v2" in Trainer.MODELS
    for model in MODEL_KINDS:
        _lib, lib, rc = _create(default_spec(model))
        assert (rc == _lib.SRS_ERR_INVALID) == (model not in Trainer.MODELS), (model, rc, lib.srs_last_error())


def test_create_ex_names_create_any_and_keeps_its_list():
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    sp = _spec_struct(default_spec("deepfm_v2"))
    out = C.c_void_p()
    assert lib.srs_trainer_create_ex(C.byref(sp), None, 0, 0, None, C.byref(out)) == _lib.SRS_ERR_INVALID
    assert not out.value and b"srs_trainer_create_any" in lib.srs_last_error()


def test_python_trainer_and_surface_accept_deepfm_v2():
    import inspect
    from tfrecmodel import deepfm_v2
    params = inspect.signature(deepfm_v2.fit).parameters
    assert {"epochs", "batch_size", "seed", "validation_data", "validation_split", "validation_freq"} <= set(params)
    from sparrowrecsys_b200.tfrecmodel._surface import Surface
    with pytest.raises(RuntimeError, match="load"):            # DeepFM_v2 fits, from the weights of a loaded model
        Surface("deepfm_v2").fit({"movieId": np.zeros(1, np.int32)})
