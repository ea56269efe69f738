"""GPU checks of Wide&Deep's `fit` (csrc/widendeep_train.cu and the trainer in csrc/trainer.cu, DESIGN.md section
4.18) against the float64 / float32 oracle (oracle/widendeep_train.py) and the reference script's end-to-end known
answer (tests/golden/widendeep_fit.json)."""
import json
import os

import numpy as np
import pytest

from oracle import widendeep_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SPREAD_MULTIPLE = 4.0          # GPU-to-float64 distance allowed, in units of the float32-to-float64 distance
# tests/test_tensor_core_precision.py's embmlp_tc_kernel<wide&deep> cases allow 2e-4 on the logit, with every weight
# rounded to 16 significant bits so that it splits exactly into bf16 hi + lo; trained weights are not rounded, and a
# model trained 167 steps at E = 10 lands at 4.5e-4 on an H100, so trained models are held to 1e-3
WD_TC_LOGIT_TOL = 0.001
CUDACORE = {"embmlp_impl": "cudacore"}


def _load(part):
    base = dict(np.load(os.path.join(GOLDEN, "deepfm_trainset.npz" if part == "train" else "dien_testset.npz")))
    extra = np.load(os.path.join(GOLDEN, "widendeep_samples.npz"))
    base.update({k[len(part) + 1:]: extra[k] for k in extra.files if k.startswith(part + "_")})
    return base


@pytest.fixture(scope="module")
def trainset():
    return _load("train")


@pytest.fixture(scope="module")
def testset():
    return _load("test")


def _rows(ts, n, one_movie=False):
    """n rows of the training set, the first three of them rows without a userGenre5 (when n allows)."""
    missing = np.flatnonzero(ts["userGenre5"] < 0)
    k = min(3, n - 1)
    rest = np.setdiff1d(np.arange(n + k), missing[:k])[: n - k]
    idx = np.concatenate([missing[:k], rest]).astype(np.int64)
    f = {key: np.ascontiguousarray(v[idx]) for key, v in ts.items()}
    if one_movie:
        f["movieId"] = np.full(n, int(f["movieId"][0]), np.int32)
    return f


# (batch size, rows, epochs): 1, 2, 10 and 100 steps per batch size, the last batch partial where the rows allow
CASES = [(1, 1, 1), (1, 2, 1), (1, 5, 2), (1, 20, 5),
         (12, 7, 1), (12, 20, 1), (12, 115, 1), (12, 1190, 1),
         (33, 33, 1), (33, 50, 1), (33, 320, 1), (33, 3280, 1),
         (4096, 4096, 1), (4096, 5000, 1), (4096, 20000, 2), (4096, 40000, 10)]


def _steps(B, n, epochs):
    return epochs * -(-n // B)


def _parity(spec, f, B, epochs):
    """Every weight against the float64 oracle.  The reference shape starts from the script's own initialisers
    (for_test=False): with init_weights' larger test scale, the raw numerics (ratings counts up to 14 617, release
    years) put 4096-row steps in a regime where the float32 oracle itself strays 0.03 from float64 within 100 steps."""
    from sparrowrecsys_b200.training import Trainer
    n = len(f["label"])
    W0 = init_weights(spec, 3, for_test=False)
    orders = widendeep_train.epoch_orders(n, epochs, 11)
    args = (W0, widendeep_train.Rows.from_features(f), f["label"], orders, B)
    W64, _, _, _ = widendeep_train.fit(*args, dtype=np.float64)
    W32, _, _, _ = widendeep_train.fit(*args, dtype=np.float32)
    with Trainer(spec, W0) as tr:
        tr.fit(f, epochs=epochs, batch_size=B, order=orders)
        assert tr.iterations == _steps(B, n, epochs)
        Wg = tr.weights()
    bad = []
    for k in W0:
        assert Wg[k].shape == W0[k].shape, k
        spread = float(np.abs(W32[k] - W64[k]).max())
        err = float(np.abs(Wg[k].astype(np.float64) - W64[k]).max())
        moved = float(np.abs(W64[k] - W0[k]).max())
        ulp = float(np.spacing(np.float32(np.abs(W64[k]).max())))   # no float32 result is nearer than this
        if k == "dense_2/bias":                  # every row's dz reaches it; a table no batch row selects (a
            assert moved > 0, k                  # missing genre) or one behind a dead unit stays put, and must then
        if not err <= SPREAD_MULTIPLE * spread + ulp:   # stay put on the device too (spread 0: within one ulp)
            bad.append((k, err, spread, ulp, err / max(spread, 1e-30)))
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,epochs", CASES)
def test_short_horizon_parity(trainset, B, n, epochs):
    assert _steps(B, n, epochs) in (1, 2, 10, 100)
    _parity(default_spec("widendeep"), _rows(trainset, n), B, epochs)


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,epochs", [(33, 66, 1), (12, 40, 3)])
def test_parity_batch_of_one_movie(trainset, B, n, epochs):
    """Every row of a batch shares one movie, so the movie row takes the whole batch's gradient."""
    _parity(default_spec("widendeep"), _rows(trainset, n, one_movie=True), B, epochs)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 700])
def test_step_forward_is_the_serving_forward(trainset, n):
    """One step over all n rows in file order: the history (computed on the step's outputs before its update) is
    the cudacore kernel's evaluate of the same rows in one batch, number for number."""
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("widendeep")
    W0 = init_weights(spec, 8, for_test=False)
    f = _rows(trainset, n)
    with Trainer(spec, W0) as tr:
        h = tr.fit(f, epochs=1, batch_size=n, order=[np.arange(n)])
    with CTRModel(spec, W0, options=CUDACORE) as m:
        assert m.kernel_name == "embmlp_kernel<wide&deep>"
        loss, acc, roc, pr = m.evaluate(f, batch_size=n)
    assert (h["loss"][0], h["accuracy"][0], h["auc"][0], h["auc_1"][0]) == (loss, acc, roc, pr)


@pytest.mark.gpu
@pytest.mark.parametrize("E,hidden", [(10, (128, 128)), (64, (17, 33)), (13, (127, 1))])
def test_trainer_evaluate_is_the_rebuilt_models(trainset, testset, E, hidden):
    """Trainer.evaluate after a fit is the evaluate of a CTRModel built from the exported weights: the trainer's
    arrays hold the weights where build_embmlp puts them, and get_weights inverts the row map and the padding."""
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("widendeep", emb_dim=E, hidden=hidden)
    f = _rows(trainset, 500)
    test = {k: v[:900] for k, v in testset.items()}
    with Trainer(spec, init_weights(spec, 2, for_test=False)) as tr:
        tr.fit(f, epochs=1, batch_size=12, seed=3)
        got = tr.evaluate(test)
        W = tr.weights()
    with CTRModel(spec, W, options=CUDACORE) as m:
        assert m.evaluate(test, batch_size=900) == got


@pytest.mark.gpu
def test_fit_is_deterministic(trainset):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("widendeep")
    W0 = init_weights(spec, 4, for_test=False)
    f = _rows(trainset, 5000)
    outs = []
    for _ in range(2):
        with Trainer(spec, W0) as tr:
            h = tr.fit(f, epochs=2, batch_size=33, seed=5)
            outs.append((h, tr.weights()))
    assert outs[0][0] == outs[1][0]
    for k in W0:
        assert np.array_equal(outs[0][1][k], outs[1][1][k]), k


@pytest.mark.gpu
def test_validation_is_evaluate_after_each_epoch_and_changes_nothing(trainset, testset):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("widendeep")
    W0 = init_weights(spec, 5, for_test=False)
    f = _rows(trainset, 800)
    val = {k: v[:400] for k, v in testset.items()}
    orders = widendeep_train.epoch_orders(800, 2, 4)
    with Trainer(spec, W0) as a:
        ha = a.fit(f, epochs=2, batch_size=12, order=orders, validation_data=val)
        Wa, ita = a.weights(), a.iterations
    with Trainer(spec, W0) as b:
        hb = b.fit(f, epochs=2, batch_size=12, order=orders)
        assert b.iterations == ita
        assert all(np.array_equal(Wa[k], b.weights()[k]) for k in W0)
    assert {k: ha[k] for k in hb} == hb
    with Trainer(spec, W0) as c:                              # one epoch per fit: the same bits, evaluated each time
        for e in range(2):
            c.fit(f, epochs=1, batch_size=12, order=orders[e:e + 1])
            loss, acc, roc, pr = c.evaluate(val)
            assert (ha["val_loss"][e], ha["val_accuracy"][e], ha["val_auc"][e], ha["val_auc_1"][e]) == \
                (loss, acc, roc, pr)
        assert all(np.array_equal(Wa[k], c.weights()[k]) for k in W0)


@pytest.mark.gpu
def test_rejected_fit_leaves_the_trainer_unchanged(trainset):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("widendeep")
    f = _rows(trainset, 100)
    at = np.arange(100)
    with Trainer(spec, init_weights(spec, 7, for_test=False)) as tr:
        tr.fit(f, epochs=1, batch_size=12, seed=0)
        before, it = tr.weights(), tr.iterations
        bad_genre = dict(f, userGenre4=np.where(at == 40, 19, f["userGenre4"]).astype(np.int32))
        bad_rated = dict(f, userRatedMovie1=np.where(at == 99, 1001, f["userRatedMovie1"]).astype(np.int32))
        bad_label = dict(f, label=np.where(at == 50, 2, f["label"]).astype(np.int32))
        no_genre = {k: v for k, v in f.items() if k != "movieGenre3"}
        dup = widendeep_train.epoch_orders(100, 2, 0)
        dup[1, 5] = dup[1, 6]
        with pytest.raises(ValueError, match="[Gg]enre"):
            tr.fit(bad_genre, epochs=1)
        with pytest.raises(ValueError, match="userRatedMovie1|history"):
            tr.fit(bad_rated, epochs=1)
        with pytest.raises(ValueError, match="label"):
            tr.fit(bad_label, epochs=1)
        with pytest.raises(KeyError, match="movieGenre3"):
            tr.fit(no_genre, epochs=1)
        with pytest.raises(ValueError, match="permutation"):
            tr.fit(f, epochs=2, order=dup)
        assert tr.iterations == it
        after = tr.weights()
        assert all(np.array_equal(before[k], after[k]) for k in before)
        tr.fit(f, epochs=1, batch_size=12, seed=0)                  # and it still trains
        assert tr.iterations == it + 9


@pytest.mark.gpu
def test_abi_rejects_a_bad_genre_or_rated_movie_before_any_launch(trainset):
    """The library's own checks, past encode_batch: a genre index >= n_genres in any slot or a userRatedMovie1
    outside the movies is SRS_ERR_RANGE, a missing history SRS_ERR_INVALID, and the trainer is unchanged."""
    import ctypes as C
    from sparrowrecsys_b200 import _lib
    from sparrowrecsys_b200.features import encode_batch
    from sparrowrecsys_b200.model import _host_struct
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("widendeep")
    f = _rows(trainset, 50)
    with Trainer(spec, init_weights(spec, 9, for_test=False)) as tr:
        before = tr.weights()
        lab = np.ascontiguousarray(f["label"], np.int32)
        order = np.arange(50, dtype=np.int32)

        def fit_with(edit_enc=lambda enc: None, edit_b=lambda b: None):
            enc = encode_batch(spec, f)
            edit_enc(enc)
            keep = []
            b = _host_struct(enc, keep)
            edit_b(b)
            return tr._lib.srs_trainer_fit_host(tr._h, C.byref(b), lab.ctypes.data, order.ctypes.data, 12, 1, None)

        for col, j, name in (("movie_genre", 2, b"movieGenre3"), ("user_genre", 4, b"userGenre5")):
            rc = fit_with(lambda enc: getattr(enc, col).__setitem__((7, j), 19))
            assert rc == _lib.SRS_ERR_RANGE and name in tr._lib.srs_last_error()
        rc = fit_with(lambda enc: enc.hist.__setitem__((3, 0), 1001))
        assert rc == _lib.SRS_ERR_RANGE and b"userRatedMovie1" in tr._lib.srs_last_error()
        rc = fit_with(edit_b=lambda b: setattr(b, "hist", None))
        assert rc == _lib.SRS_ERR_INVALID
        assert tr.iterations == 0
        after = tr.weights()
        assert all(np.array_equal(before[k], after[k]) for k in before)


def _band(fit):
    """The seed-to-seed band of the oracle's test metrics, widened by half its width on each side (as NeuralCF's)."""
    out = {}
    for k, (lo, hi) in fit["band"].items():
        w = hi - lo
        out[k] = (lo - w / 2, hi + w / 2)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("E", [10, 32])
def test_trained_model_serves(trainset, testset, E):
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("widendeep", emb_dim=E)
    with Trainer(spec, init_weights(spec, 6, for_test=False)) as tr:
        tr.fit(_rows(trainset, 2000), epochs=1, batch_size=12, seed=1)
        W = tr.weights()
        m = tr.to_model()
    f = {k: v[-300:] for k, v in testset.items()}
    po, zo, _ = widendeep_train.forward(W, widendeep_train.Rows.from_features(f), np.float64)
    with CTRModel(spec, W, options=CUDACORE) as mc:
        pc = mc.predict(f)
    assert np.abs(pc[:, 0] - po).max() <= 2e-6
    p, z = m.predict_with_logits(f)
    if E <= 12:                                   # the default kernel at E <= 12 is the tensor-core one
        assert m.kernel_name == "embmlp_tc_kernel<wide&deep>"
        assert np.abs(z[:, 0] - zo).max() <= WD_TC_LOGIT_TOL
        assert np.abs(p[:, 0] - po).max() <= WD_TC_LOGIT_TOL / 4
    else:
        assert np.abs(p[:, 0] - po).max() <= 2e-6
    m.close()


@pytest.mark.gpu
def test_the_script_end_to_end(trainset, testset):
    """WideNDeep.py: an untrained model, fit(train, epochs=5) at batch 12, then evaluate on testSamples."""
    from tfrecmodel import widendeep
    with open(os.path.join(GOLDEN, "widendeep_fit.json")) as fh:
        fit = json.load(fh)
    widendeep.load(seed=0)
    hist = widendeep.fit(trainset, epochs=5, batch_size=12, seed=0)
    assert len(hist["loss"]) == 5
    loss, acc, roc, pr = widendeep.evaluate(testset, batch_size=12)
    band = _band(fit)
    got = {"loss": loss, "accuracy": acc, "roc_auc": roc, "pr_auc": pr}
    print("widendeep end to end:", got, "band", fit["band"])
    for k, (lo, hi) in band.items():
        assert lo <= got[k] <= hi, (k, got[k], band[k])
    oracle0 = fit["runs"][0]["history"]
    # the training history follows the oracle's seed-0 run closely in the first epoch
    assert abs(hist["loss"][0] - oracle0[0]["loss"]) < 5e-3
    assert abs(hist["auc"][0] - oracle0[0]["roc_auc"]) < 5e-3
    p = widendeep.predict({k: v[:4] for k, v in testset.items()})
    assert p.shape == (4, 1)
