"""CPU checks of Wide&Deep `fit`'s oracle (oracle/widendeep_train.py), its fixtures, the step kernel's dispatch and
the trainer ABI's up-front rejections for Wide&Deep (DESIGN.md section 4.18)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import ctr_oracle, keras_eval, ncf_train, widendeep_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def small_case(seed, B, hidden=(6, 5), E=3, Vm=7, Vu=9, cb=5):
    """A small Wide&Deep with repeated ids, missing genres in every slot and rows sharing a crossed bucket, at
    scales where the relus switch on both sides."""
    spec = default_spec("widendeep", emb_dim=E, n_movies=Vm, n_users=Vu, hidden=hidden, cross_buckets=cb)
    G = spec.n_genres
    W = {k: v.astype(np.float64) for k, v in init_weights(spec, seed, for_test=True).items()}
    rng = np.random.default_rng(seed + 100)
    for k in W:
        W[k] = W[k] * 2.0 + (rng.normal(0, 0.3, W[k].shape) if k.endswith("bias") else 0)
    mid = rng.integers(0, Vm, B)
    uid = rng.integers(0, Vu, B)
    mg = rng.integers(-1, G, (B, 3))
    ug = rng.integers(-1, G, (B, 5))
    rated = rng.integers(0, Vm, B)
    mid[: B // 2] = mid[0]                                    # repeated ids
    mg[: B // 3, 1] = mg[0, 1]
    if B > 1:
        rated[1], mid[1] = rated[0], mid[0]                   # two rows on one crossed bucket
    mg[-1, :] = -1                                            # the last row misses every genre
    ug[-1, :] = -1
    num = rng.normal(0, 1, (B, 7)).astype(np.float32)
    y = rng.integers(0, 2, B)
    return spec, W, widendeep_train.Rows(mid, uid, mg, ug, num, rated), y


@pytest.mark.parametrize("seed,B", [(0, 12), (1, 33)])
def test_forward_is_ctr_oracle_widendeep_forward(seed, B):
    spec, W, r, _ = small_case(seed, B)
    p, z, _ = widendeep_train.forward(W, r, np.float64)
    po, zo = ctr_oracle.widendeep_forward(spec, W, r.features(), np.float64)
    np.testing.assert_allclose(z, zo[:, 0], rtol=0, atol=1e-12)
    np.testing.assert_allclose(p, po[:, 0], rtol=0, atol=1e-12)


def _load(part):
    base = dict(np.load(os.path.join(GOLDEN, "deepfm_trainset.npz" if part == "train" else "dien_testset.npz")))
    extra = np.load(os.path.join(GOLDEN, "widendeep_samples.npz"))
    base.update({k[len(part) + 1:]: extra[k] for k in extra.files if k.startswith(part + "_")})
    return base


def test_forward_on_the_testset_is_ctr_oracle_widendeep_forward():
    spec = default_spec("widendeep")
    W = init_weights(spec, 1, for_test=False)
    f = {k: v[:2000] for k, v in _load("test").items()}
    assert (f["userGenre5"] < 0).any()
    _, z, _ = widendeep_train.forward(W, widendeep_train.Rows.from_features(f), np.float64)
    _, zo = ctr_oracle.widendeep_forward(spec, W, f, np.float64)
    np.testing.assert_allclose(z, zo[:, 0], rtol=0, atol=1e-12)


@pytest.mark.parametrize("seed,B", [(0, 1), (1, 5), (2, 12)])
def test_backward_matches_central_differences(seed, B):
    _, W, r, y = small_case(seed, B)
    g, _, _ = widendeep_train.gradients(W, r, y, np.float64)
    h = 1e-6
    for name, w in W.items():
        num = np.zeros_like(w)
        for i in np.ndindex(w.shape):
            old = w[i]
            w[i] = old + h
            lp = widendeep_train.batch_loss(W, r, y)
            w[i] = old - h
            lm = widendeep_train.batch_loss(W, r, y)
            w[i] = old
            num[i] = (lp - lm) / (2 * h)
        np.testing.assert_allclose(g[name], num, rtol=1e-5, atol=1e-8, err_msg=name)


def test_missing_genres_give_no_gradient_and_shared_buckets_add_up():
    _, W, r, y = small_case(3, 6)
    r.mg[:] = -1
    r.ug[:] = -1
    g, _, _ = widendeep_train.gradients(W, r, y, np.float64)
    for name in widendeep_train.MOVIE_GENRES + widendeep_train.USER_GENRES:
        assert not g[name].any(), name
    assert g["movieId_embedding"].any() and g["userId_embedding"].any()
    # rows 0 and 1 share a bucket: its wide row's gradient is the sum of their dz
    p, _, c = widendeep_train.forward(W, r, np.float64)
    dz = (p - y) / len(y)
    b = c["bucket"]
    assert b[0] == b[1]
    h1 = W["dense_1/kernel"].shape[1]
    np.testing.assert_allclose(g["dense_2/kernel"][h1 + b[0], 0], dz[b == b[0]].sum(), rtol=1e-12)


def test_partial_last_batch_divides_by_its_own_size():
    _, W, r, y = small_case(4, 12)
    order = np.arange(12)[None, :]
    W5, _, _, _ = widendeep_train.fit(W, r, y, order, 5, np.float64, max_steps=2)
    g, _, _ = widendeep_train.gradients(W5, r.take(np.arange(10, 12)), y[10:], np.float64)
    g2 = [widendeep_train.gradients(W5, r.take(np.array([i])), y[i:i + 1], np.float64)[0] for i in (10, 11)]
    for k in g:
        np.testing.assert_allclose(g[k], (g2[0][k] + g2[1][k]) / 2, rtol=1e-12, atol=1e-15, err_msg=k)


def test_adam_first_step_moves_each_parameter_by_lr_sign_g():
    _, W, r, y = small_case(5, 12)
    g, _, _ = widendeep_train.gradients(W, r, y, np.float64)
    W1 = {k: v.copy() for k, v in W.items()}
    widendeep_train.Adam(W1, np.float64).step(W1, g)
    for k in W:
        d = W1[k] - W[k]
        np.testing.assert_allclose(d, -0.001 * g[k] / (np.abs(g[k]) + 1e-7 / np.sqrt(0.001)), rtol=1e-9,
                                   atol=1e-18, err_msg=k)
        assert np.all(d[g[k] == 0] == 0), k


def _two_steps(W, r, y, lazy):
    orders = np.array([np.arange(len(y))])
    W1, _, _, _ = widendeep_train.fit(W, r, y, orders, 2, np.float64, lazy=lazy, max_steps=1)
    W2, _, _, _ = widendeep_train.fit(W, r, y, orders, 2, np.float64, lazy=lazy, max_steps=2)
    return W1, W2


def _moved_by_decay(G):
    """What a parameter with step-1 gradient G and no step-2 gradient moves by at step 2 (m = 0.09 G,
    v = 0.000999 G^2 under either form)."""
    alpha = 0.001 * np.sqrt(1 - 0.999 ** 2) / (1 - 0.9 ** 2)
    return -alpha * (0.9 * 0.1 * G) / (np.sqrt(0.999 * 0.001 * G * G) + 1e-7)


def _absent_case(seed):
    """Four rows: step 1 (rows 0, 1) has movie 1, genre 4 in movieGenre2 and a wide bucket step 2 lacks."""
    spec, W, r, y = small_case(seed, 4, cb=97)
    r.mid[:] = [1, 1, 2, 3]
    r.rated[:] = [0, 0, 5, 6]
    r.mg[:, 1] = [4, 4, -1, 2]
    b = r.bucket(97)
    assert b[0] not in b[2:]
    return spec, W, r, y


def test_wide_row_absent_from_step_two_moves_by_the_dense_form():
    """dense_2/kernel is a dense variable (the crossed column's one-hot is a dense input, so its gradient is a MatMul
    gradient): a wide row of the step-1 batch that step 2 does not hit still moves at step 2, lazy or not."""
    _, W, r, y = _absent_case(6)
    g1, _, _ = widendeep_train.gradients(W, r.take(np.arange(2)), y[:2], np.float64)
    row = W["dense_1/kernel"].shape[1] + r.bucket(97)[0]
    expect = _moved_by_decay(g1["dense_2/kernel"][row, 0])
    for lazy in (False, True):
        W1, W2 = _two_steps(W, r, y, lazy)
        moved = W2["dense_2/kernel"][row, 0] - W1["dense_2/kernel"][row, 0]
        np.testing.assert_allclose(moved, expect, rtol=1e-9)
        assert abs(moved) > 1e-4


def test_table_rows_absent_from_step_two_move_by_the_sparse_form_and_lazy_adam_differs():
    _, W, r, y = _absent_case(7)
    g1, _, _ = widendeep_train.gradients(W, r.take(np.arange(2)), y[:2], np.float64)
    moved, final = {}, {}
    for lazy in (False, True):
        W1, W2 = _two_steps(W, r, y, lazy)
        moved[lazy] = {"movieId_embedding": W2["movieId_embedding"][1] - W1["movieId_embedding"][1],
                       "movieGenre2_embedding": W2["movieGenre2_embedding"][4] - W1["movieGenre2_embedding"][4]}
        final[lazy] = W2
    for k in moved[False]:
        row = 1 if k == "movieId_embedding" else 4
        np.testing.assert_allclose(moved[False][k], _moved_by_decay(g1[k][row]), rtol=1e-9, err_msg=k)
        assert np.all(np.abs(moved[False][k]) > 1e-4), k
        assert np.all(moved[True][k] == 0), k
    assert not np.array_equal(final[False]["movieId_embedding"], final[True]["movieId_embedding"])
    # the sparse form itself on a Wide&Deep table: m = b1 m + (1 - b1) g
    opt = widendeep_train.Adam({"userGenre5_embedding": np.zeros(1)}, np.float64)
    opt.m["userGenre5_embedding"][0] = 0.3
    opt.step({"userGenre5_embedding": np.zeros(1)}, {"userGenre5_embedding": np.zeros(1)})
    assert opt.m["userGenre5_embedding"][0] == 0.9 * 0.3 + (1 - 0.9) * 0


def test_float32_oracle_tracks_float64():
    _, W, r, y = small_case(8, 40)
    orders = widendeep_train.epoch_orders(40, 2, 7)
    W64, h64, _, _ = widendeep_train.fit(W, r, y, orders, 12, np.float64)
    W32, h32, _, _ = widendeep_train.fit(W, r, y, orders, 12, np.float32)
    for k in W:
        assert np.abs(W32[k] - W64[k]).max() < 1e-5, k
    assert abs(h32[-1]["loss"] - h64[-1]["loss"]) < 1e-5


def test_fit_validate_is_fit_plus_evaluate_after_the_validated_epochs():
    """widendeep_train.fit_validate: the training of `fit`, bit for bit; the validated epochs' forward of the
    validation rows; epoch by epoch with the carried Adam state gives one call's bits (fit_validation.fit's rules)."""
    _, W, r, y = small_case(9, 30)
    f = dict(r.features(), label=y)
    _, _, rv, yv = small_case(10, 20)
    val = dict(rv.features(), label=yv)
    orders = widendeep_train.epoch_orders(30, 4, 3)
    Wa, ha, va, _ = widendeep_train.fit_validate(W, f, orders, 12, np.float64, val=val, validation_freq=2)
    Wb, hb, _, _ = widendeep_train.fit(W, r, y, orders, 12, np.float64)
    assert ha == hb
    assert all(np.array_equal(Wa[k], Wb[k]) for k in W)
    assert va[0] is None and va[2] is None
    p, z, _ = widendeep_train.forward(Wa, rv, np.float64)
    r = keras_eval.keras_evaluate(p.astype(np.float32), z.astype(np.float32), yv)
    assert va[3] == {k: r[k] for k in ("loss", "accuracy", "roc_auc", "pr_auc")}
    Wc, opt = W, None
    for e in range(4):
        Wc, _, vc, opt = widendeep_train.fit_validate(Wc, f, orders[e:e + 1], 12, np.float64, val=val, opt=opt)
        if e % 2 == 1:
            assert vc[0] == va[e]
    assert all(np.array_equal(Wa[k], Wc[k]) for k in W)


# ---- what the GPU parity tolerance detects ----------------------------------------------------------------------
MULTIPLE = 4.0          # tests/test_gpu_fit_widendeep.py's SPREAD_MULTIPLE


def _mutant(kind):
    """widendeep_train.gradients with one deliberate mistake."""
    base = widendeep_train.gradients

    def g(W, r, y, dtype=np.float32):
        if kind == "row":                                     # a dropped batch row (the last, when B > 1)
            _, p, z = base(W, r, y, dtype)
            if len(y) > 1:
                out, _, _ = base(W, r.take(np.arange(len(y) - 1)), y[:-1], dtype)
                scale = dtype((len(y) - 1) / len(y))
                return {k: v * scale for k, v in out.items()}, p, z
            return base(W, r, y, dtype)
        out, p, z = base(W, r, y, dtype)
        if kind == "column":                                  # a dropped embedding column
            out["userGenre3_embedding"][...] = 0
        elif kind == "hidden":                                # a dropped hidden unit of the first layer
            out["dense/kernel"][:, 0] = 0
            out["dense/bias"][0] = 0
        elif kind == "wide":                                  # a dropped wide entry (the first row's)
            h1 = W["dense_1/kernel"].shape[1]
            _, _, c = widendeep_train.forward(W, r, dtype)
            b = c["bucket"][0]
            out["dense_2/kernel"][h1 + b, 0] -= out["dense_2/kernel"][h1 + b, 0] * dtype(1 / max(1, (c["bucket"] == b).sum()))
        return out, p, z
    return g


@pytest.mark.parametrize("B,n,epochs", [(12, 115, 1), (33, 320, 1)])
def test_parity_tolerance_detects_each_mistake(monkeypatch, B, n, epochs):
    spec = default_spec("widendeep")
    W0 = init_weights(spec, 3, for_test=False)                  # as the GPU parity cases of the reference shape
    f = {k: v[:n] for k, v in _load("train").items()}
    rows = widendeep_train.Rows.from_features(f)
    orders = widendeep_train.epoch_orders(n, epochs, 11)
    args = (W0, rows, f["label"], orders, B)
    W64, _, _, _ = widendeep_train.fit(*args, dtype=np.float64)
    W32, _, _, _ = widendeep_train.fit(*args, dtype=np.float32)

    def tol(k):
        return MULTIPLE * float(np.abs(W32[k] - W64[k]).max()) + float(np.spacing(np.float32(np.abs(W64[k]).max())))

    for k in W0:
        assert np.abs(W64[k] - W0[k]).max() > tol(k), k       # every tensor moves past its tolerance
    caught = {}
    for kind in ("column", "hidden", "row", "wide"):
        monkeypatch.setattr(widendeep_train, "gradients", _mutant(kind))
        Wm, _, _, _ = widendeep_train.fit(*args, dtype=np.float64)
        monkeypatch.undo()
        caught[kind] = [k for k in W0 if np.abs(Wm[k] - W64[k]).max() > tol(k)]
    Wl, _, _, _ = widendeep_train.fit(*args, dtype=np.float64, lazy=True)
    caught["lazy"] = [k for k in W0 if np.abs(Wl[k] - W64[k]).max() > tol(k)]
    for kind, names in caught.items():
        assert names, kind


def test_train_fixtures():
    z = np.load(os.path.join(GOLDEN, "widendeep_samples.npz"))
    genres = ("movieGenre2", "movieGenre3", "userGenre2", "userGenre3", "userGenre4", "userGenre5")
    assert sorted(z.files) == sorted(["train_%s" % g for g in genres] + ["test_%s" % g for g in genres]
                                     + ["train_userRatedMovie1"])
    for k in z.files:
        n = 88827 if k.startswith("train_") else 22440
        assert z[k].shape == (n,), k
        if "Genre" in k:
            assert z[k].dtype == np.int8 and z[k].min() >= -1 and z[k].max() < 19, k
    assert z["train_userRatedMovie1"].dtype == np.int32
    assert 0 <= z["train_userRatedMovie1"].min() and z["train_userRatedMovie1"].max() < 1001
    with open(os.path.join(GOLDEN, "widendeep_fit.json")) as f:
        fit = json.load(f)
    assert fit["rows"] == 88827 and fit["test_rows"] == 22440 and fit["epochs"] == 5 and fit["batch_size"] == 12
    assert [r["seed"] for r in fit["runs"]] == fit["seeds"] and 0 in fit["seeds"]
    for r in fit["runs"]:
        assert r["iterations"] == 5 * 7403 and len(r["history"]) == 5 and r["oracle_seconds"] > 0
        for k, (lo, hi) in fit["band"].items():
            assert lo <= r["test"][k] <= hi


@pytest.mark.skipif(not os.path.exists("/root/reference/src/main/resources/webroot/sampledata/trainingSamples.csv"),
                    reason="needs the reference checkout")
def test_generator_reproduces_the_columns():
    import subprocess
    import sys
    subprocess.check_call([sys.executable, os.path.join(GOLDEN, "make_widendeep_train_golden.py"), "--check"])


# ---- the trainer ABI's rejections that need no device ----------------------------------------------------------
def _lib_or_skip():
    from sparrowrecsys_b200 import _lib
    try:
        return _lib, _lib.load()
    except ImportError as e:
        pytest.skip(str(e))


def _create(spec, hp=None, **fields):
    """srs_trainer_create_ex with no tensors; `fields` override the srs_spec struct (shapes ModelSpec refuses)."""
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    sp = _spec_struct(spec)
    for k, v in fields.items():
        setattr(sp, k, v)
    out = C.c_void_p()
    rc = lib.srs_trainer_create_ex(C.byref(sp), None, 0, 0, None if hp is None else C.byref(hp), C.byref(out))
    assert not out.value
    return _lib, lib, rc


@pytest.mark.parametrize("overrides,match", [(dict(hidden=(129, 128)), b"1..128"), (dict(hidden=(128, 129)), b"1..128"),
                                             (dict(hidden=(0, 128)), b"1..128"),
                                             (dict(hidden=(128, 128, 128)), b"exactly 2"),
                                             (dict(hidden=(128,)), b"exactly 2")])
def test_trainer_rejects_unsupported_widendeep_shapes(overrides, match):
    _lib, lib, rc = _create(default_spec("widendeep", **overrides))
    assert rc == _lib.SRS_ERR_INVALID and match in lib.srs_last_error()


def test_trainer_rejects_widendeep_emb_dim_65_and_no_buckets():
    _lib, lib, rc = _create(default_spec("widendeep", emb_dim=64), emb_dim=65)
    assert rc == _lib.SRS_ERR_INVALID and b"emb_dim" in lib.srs_last_error()
    _lib, lib, rc = _create(default_spec("widendeep"), cross_buckets=0)
    assert rc == _lib.SRS_ERR_INVALID and b"cross_buckets" in lib.srs_last_error()


@pytest.mark.parametrize("hp", [dict(lr=0.0), dict(beta_1=1.0), dict(beta_2=-0.1), dict(epsilon=0.0)])
def test_trainer_rejects_bad_adam_hyperparameters_for_widendeep(hp):
    _lib, _ = _lib_or_skip()
    a = _lib.SrsAdam(**dict(ncf_train.KERAS_ADAM, **hp))
    _lib, lib, rc = _create(default_spec("widendeep"), a)
    assert rc == _lib.SRS_ERR_INVALID


def test_trainer_create_ex_still_rejects_models_without_fit():
    for model in ("embeddingmlp", "deepfm_v2", "dien", "din", "twotowers"):
        _lib, lib, rc = _create(default_spec(model))
        assert rc == _lib.SRS_ERR_INVALID
        msg = lib.srs_last_error()
        assert b"NeuralCF" in msg and b"DeepFM" in msg and b"Wide&Deep" in msg


def test_trainer_create_keeps_its_two_models_and_names_the_ex_entry_point():
    """srs_trainer_create's documented list (NeuralCF, DeepFM) is unchanged: Wide&Deep goes through
    srs_trainer_create_ex, and srs_trainer_create's message says so."""
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    sp = _spec_struct(default_spec("widendeep"))
    out = C.c_void_p()
    assert lib.srs_trainer_create(C.byref(sp), None, 0, 0, None, C.byref(out)) == _lib.SRS_ERR_INVALID
    assert not out.value and b"srs_trainer_create_ex" in lib.srs_last_error()
    sp.hidden[0] = 129                                 # the same spec through _ex reaches Wide&Deep's own checks
    assert lib.srs_trainer_create_ex(C.byref(sp), None, 0, 0, None, C.byref(out)) == _lib.SRS_ERR_INVALID
    assert b"Wide&Deep's hidden widths" in lib.srs_last_error()


def test_python_trainer_and_surface_accept_widendeep():
    import inspect
    from sparrowrecsys_b200.training import Trainer
    from tfrecmodel import widendeep
    assert "widendeep" in Trainer.MODELS and "embeddingmlp" not in Trainer.MODELS
    with pytest.raises(NotImplementedError, match="Wide&Deep"):
        Trainer(default_spec("embeddingmlp"), {})
    params = inspect.signature(widendeep.fit).parameters
    assert {"epochs", "batch_size", "seed", "validation_data", "validation_split", "validation_freq"} <= set(params)
    from sparrowrecsys_b200.tfrecmodel._surface import Surface
    with pytest.raises(RuntimeError, match="load"):            # Wide&Deep fits, from the weights of a loaded model
        Surface("widendeep").fit({"movieId": np.zeros(1, np.int32)})
