"""GPU checks of the two-tower model's `fit` (neural_cf_model_2 with its final Dense; csrc/twotowers_train.cu,
csrc/trainer.cu, DESIGN.md section 4.27) against the float64 / float32 oracle (oracle/twotowers_train.py), at every
step instantiation of `TT_MATRIX` (tests/test_fit_oracle_twotowers.py), and end to end against the golden band of
the script's run (tests/golden/twotowers_fit.json)."""
import json
import os

import numpy as np
import pytest

from oracle import keras_eval, ncf_train, twotowers_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights
from test_fit_oracle_twotowers import (GOLDEN, SPREAD_MULTIPLE, TT_MATRIX, case_id, case_spec, inputs, oracle,
                                       steps, trainset)

SERVING_KERNEL = "ncf_kernel<two_towers>"


def script_spec(**over):
    """NeuralCF.py's neural_cf_model_2 with its hidden_units [10, 10], E = 10 and the final Dense."""
    return default_spec("twotowers", **dict(dict(hidden=(10, 10), final_dense=True), **over))


def _rows(n, one_movie=False):
    f = {k: np.ascontiguousarray(v[:n]) for k, v in trainset().items()}
    if one_movie:
        f["movieId"] = np.full(n, int(f["movieId"][0]), np.int32)
    return f


def _trainer(spec, W, adam=None):
    from sparrowrecsys_b200.training import Trainer
    return Trainer(spec, W, adam=adam)


def _check_parity(W0, Wg, W64, W32, tol=None):
    for k in W0:
        assert Wg[k].shape == W0[k].shape, k
        spread = float(np.abs(W32[k] - W64[k]).max())
        err = float(np.abs(Wg[k].astype(np.float64) - W64[k]).max())
        allowed = SPREAD_MULTIPLE * spread + 1e-9 if tol is None else tol[k]
        assert float(np.abs(W64[k] - W0[k]).max()) > 0, k
        assert err <= allowed, (k, err, spread, allowed)


# (batch size, rows, epochs): 1, 2, 10 and 100 steps per batch size, the last batch partial where the rows allow
CASES = [(1, 1, 1), (1, 2, 1), (1, 5, 2), (1, 20, 5),
         (12, 7, 1), (12, 20, 1), (12, 115, 1), (12, 1190, 1),
         (33, 33, 1), (33, 50, 1), (33, 320, 1), (33, 3280, 1),
         (4096, 4096, 1), (4096, 5000, 1), (4096, 20000, 2), (4096, 40000, 10)]


def _parity(B, n, epochs, one_movie):
    spec = script_spec()
    W0 = init_weights(spec, 3, for_test=True)
    f = _rows(n, one_movie)
    orders = ncf_train.epoch_orders(n, epochs, 11)
    args = (W0, f["movieId"], f["userId"], f["label"], orders, B)
    W64 = twotowers_train.fit(*args, dtype=np.float64)[0]
    W32 = twotowers_train.fit(*args, dtype=np.float32)[0]
    with _trainer(spec, W0) as tr:
        tr.fit(f, epochs=epochs, batch_size=B, order=orders)
        assert tr.iterations == epochs * -(-n // B)
        Wg = tr.weights()
    _check_parity(W0, Wg, W64, W32)


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,epochs", CASES)
def test_short_horizon_parity(B, n, epochs):
    assert epochs * -(-n // B) in (1, 2, 10, 100)
    _parity(B, n, epochs, one_movie=False)


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,epochs", [(33, 66, 1), (12, 40, 3)])
def test_parity_batch_of_one_movie(B, n, epochs):
    _parity(B, n, epochs, one_movie=True)


# ---- every step instantiation ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", TT_MATRIX, ids=case_id)
def test_trainer_exports_its_initial_weights_exactly(case):
    W0 = inputs(case)[0]
    with _trainer(case_spec(case), W0, case.adam) as tr:
        W = tr.weights()
        assert tr.iterations == 0
    assert W.keys() == W0.keys()
    for k in W0:
        assert W[k].shape == W0[k].shape and np.array_equal(W[k], W0[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", TT_MATRIX, ids=case_id)
def test_fit_matches_float64_oracle(case):
    """Every tensor within 4x the float32 oracle's spread (plus one ulp) of the float64 fit.  The cases run in
    TT_MATRIX's order in one process, so <32, 32> runs below its three-layer opt-in and then at it."""
    W0, f, orders = inputs(case)
    W64, W32, tol = oracle(case)
    with _trainer(case_spec(case), W0, case.adam) as tr:
        tr.fit(f, epochs=case.epochs, batch_size=case.B, order=orders)
        assert tr.iterations == steps(case)
        Wg = tr.weights()
    _check_parity(W0, Wg, W64, W32, tol)


@pytest.mark.gpu
@pytest.mark.parametrize("case", TT_MATRIX, ids=case_id)
def test_step_forward_is_the_serving_forward(case):
    """One step over all n rows in file order: its history (the step's outputs before its update) is the serving
    model's evaluate of the same rows in one batch, number for number."""
    from sparrowrecsys_b200.model import CTRModel
    W0, f, _ = inputs(case)
    with _trainer(case_spec(case), W0, case.adam) as tr:
        h = tr.fit(f, epochs=1, batch_size=case.n, order=[np.arange(case.n)])
    with CTRModel(case_spec(case), W0) as m:
        assert m.kernel_name == SERVING_KERNEL
        loss, acc, roc, pr = m.evaluate(f, batch_size=case.n)
    assert (h["loss"][0], h["accuracy"][0], h["auc"][0], h["auc_1"][0]) == (loss, acc, roc, pr)


@pytest.mark.gpu
@pytest.mark.parametrize("case", TT_MATRIX, ids=case_id)
def test_trainer_evaluate_is_the_rebuilt_models(case):
    """After the fit, the trainer's forward over its own padded arrays is that of a serving model built from the
    exported weights, whose padding is zero by construction."""
    from sparrowrecsys_b200.model import CTRModel
    W0, f, orders = inputs(case)
    with _trainer(case_spec(case), W0, case.adam) as tr:
        tr.fit(f, epochs=case.epochs, batch_size=case.B, order=orders)
        W = tr.weights()
        got = tr.evaluate_result(f)
    with CTRModel(case_spec(case), W) as m:
        want = m.evaluate_result(f, batch_size=case.n)
    assert got.rows == case.n
    assert (got.rows, got.positives, got.correct) == (want.rows, want.positives, want.correct)
    assert (got.loss, got.accuracy, got.roc_auc, got.pr_auc) == (want.loss, want.accuracy, want.roc_auc, want.pr_auc)


@pytest.mark.gpu
@pytest.mark.parametrize("case", TT_MATRIX, ids=case_id)
def test_fit_is_deterministic(case):
    W0, f, orders = inputs(case)
    outs = []
    for _ in range(2):
        with _trainer(case_spec(case), W0, case.adam) as tr:
            outs.append((tr.fit(f, epochs=case.epochs, batch_size=case.B, order=orders), tr.weights()))
    assert outs[0][0] == outs[1][0]
    for k in W0:
        assert np.array_equal(outs[0][1][k], outs[1][1][k]), k


# ---- the script's model ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_history_matches_keras_evaluate_of_the_oracle_steps():
    spec = script_spec()
    W0 = init_weights(spec, 5, for_test=False)
    n, B, epochs = 600, 12, 2
    f = _rows(n)
    orders = ncf_train.epoch_orders(n, epochs, 2)
    _, _, out, _ = twotowers_train.fit(W0, f["movieId"], f["userId"], f["label"], orders, B, np.float64,
                                       keep_outputs=True)
    with _trainer(spec, W0) as tr:
        h = tr.fit(f, epochs=epochs, batch_size=B, order=orders)
    per = -(-n // B)
    for e in range(epochs):
        p = np.concatenate([o[0] for o in out[e * per:(e + 1) * per]])
        z = np.concatenate([o[1] for o in out[e * per:(e + 1) * per]])
        y = np.concatenate([o[2] for o in out[e * per:(e + 1) * per]])
        r = keras_eval.keras_evaluate(p.astype(np.float32), z.astype(np.float32), y)
        assert abs(h["loss"][e] - r["loss"]) <= 1e-5, (e, h["loss"][e], r["loss"])
        assert abs(h["accuracy"][e] - r["accuracy"]) <= 2.0 / n
        assert abs(h["auc"][e] - r["roc_auc"]) <= 2e-3 and abs(h["auc_1"][e] - r["pr_auc"]) <= 2e-3


@pytest.mark.gpu
def test_trained_model_predicts_and_evaluates_as_the_trainer():
    spec = script_spec()
    t = np.load(os.path.join(GOLDEN, "neuralcf_002_testset.npz"))
    test = {"movieId": t["movieId"][:3000], "userId": t["userId"][:3000], "label": t["label"][:3000]}
    with _trainer(spec, init_weights(spec, 6, for_test=False)) as tr:
        tr.fit(_rows(2000), epochs=1, batch_size=12, seed=1)
        W = tr.weights()
        ev = tr.evaluate(test)
        m = tr.to_model()
    with m:
        assert m.kernel_name == SERVING_KERNEL
        assert m.evaluate(test) == ev
        p = m.predict({"movieId": test["movieId"], "userId": test["userId"]})
    po, _, _ = twotowers_train.forward(W, test["movieId"], test["userId"], np.float64)
    assert np.abs(p[:, 0] - po).max() <= 2e-5


@pytest.mark.gpu
def test_validation_logs_the_selected_epochs_and_changes_nothing():
    spec = script_spec()
    W0 = init_weights(spec, 8, for_test=False)
    f = _rows(1500)
    t = np.load(os.path.join(GOLDEN, "neuralcf_002_testset.npz"))
    val = {"movieId": t["movieId"][:800], "userId": t["userId"][:800], "label": t["label"][:800]}
    with _trainer(spec, W0) as plain:
        hp = plain.fit(f, epochs=3, batch_size=12, seed=4)
        Wp = plain.weights()
    with _trainer(spec, W0) as tr:
        h2 = tr.fit(f, epochs=2, batch_size=12, seed=4, validation_data=val, validation_freq=2)
        after2 = tr.evaluate(val)
    assert sorted(h2) == ["accuracy", "auc", "auc_1", "loss", "val_accuracy", "val_auc", "val_auc_1", "val_loss"]
    assert all(len(h2["val_" + k]) == 1 for k in ("loss", "accuracy", "auc", "auc_1"))   # epoch 2 only
    assert (h2["val_loss"][0], h2["val_accuracy"][0], h2["val_auc"][0], h2["val_auc_1"][0]) == after2
    with _trainer(spec, W0) as tr:
        h3 = tr.fit(f, epochs=3, batch_size=12, seed=4, validation_data=(val, val["label"]))
        Wv = tr.weights()
    assert all(len(h3["val_" + k]) == 3 for k in ("loss", "accuracy", "auc", "auc_1"))
    assert {k: h3[k] for k in hp} == hp                          # the training logs and weights are the plain fit's
    assert all(np.array_equal(Wp[k], Wv[k]) for k in Wp)
    with _trainer(spec, W0) as tr:                               # the last 300 rows held out, before any shuffle
        hs = tr.fit(f, epochs=1, batch_size=12, seed=4, validation_split=0.2)
        assert tr.iterations == -(-1200 // 12)
        assert hs["val_loss"] == [tr.evaluate({k: v[1200:] for k, v in f.items()})[0]]


@pytest.mark.gpu
def test_rejections_leave_the_trainer_unchanged():
    from sparrowrecsys_b200.training import Trainer
    spec = script_spec()
    f = _rows(100)
    with _trainer(spec, init_weights(spec, 7, for_test=False)) as tr:
        tr.fit(f, epochs=1, batch_size=12, seed=0)
        before, it = tr.weights(), tr.iterations
        bad_label = dict(f, label=np.where(np.arange(100) == 50, 2, f["label"]).astype(np.int32))
        bad_movie = dict(f, movieId=np.where(np.arange(100) == 99, 1001, f["movieId"]).astype(np.int32))
        bad_user = dict(f, userId=np.where(np.arange(100) == 0, -1, f["userId"]).astype(np.int32))
        dup = ncf_train.epoch_orders(100, 2, 0)
        dup[1, 5] = dup[1, 6]
        with pytest.raises(ValueError, match="label"):
            tr.fit(bad_label, epochs=1)
        with pytest.raises(ValueError, match="movieId"):
            tr.fit(bad_movie, epochs=1)
        with pytest.raises(ValueError, match="userId"):
            tr.fit(bad_user, epochs=1)
        with pytest.raises(ValueError, match="permutation"):
            tr.fit(f, epochs=2, order=dup)
        with pytest.raises(ValueError, match="movieId"):
            tr.fit(f, epochs=1, validation_data=bad_movie)
        raw = script_spec(final_dense=False)
        with pytest.raises(ValueError, match="final Dense"):
            Trainer(raw, init_weights(raw, 7, for_test=False))
        assert tr.iterations == it
        after = tr.weights()
        assert all(np.array_equal(before[k], after[k]) for k in before)
        tr.fit(f, epochs=1, batch_size=12, seed=0)                  # and it still trains
        assert tr.iterations == it + 9


def _band(fit):
    """The seed-to-seed band of the oracle's test metrics, widened by half its width on each side: the GPU run starts
    from seed 0's weights and order but its rounding parts ways over 37 015 steps, so it is one more draw."""
    return {k: (lo - (hi - lo) / 2, hi + (hi - lo) / 2) for k, (lo, hi) in fit["band"].items()}


@pytest.mark.gpu
def test_the_script_end_to_end():
    """neural_cf_model_2 with hidden_units [10, 10] and its final Dense, untrained, fit(train, epochs=5) at batch 12
    from seed 0, then evaluated on testSamples.csv."""
    with open(os.path.join(GOLDEN, "twotowers_fit.json")) as fh:
        fit = json.load(fh)
    spec = script_spec()
    with _trainer(spec, init_weights(spec, 0, for_test=False)) as tr:
        hist = tr.fit(trainset(), epochs=5, batch_size=12, seed=0)
        t = np.load(os.path.join(GOLDEN, "neuralcf_002_testset.npz"))
        loss, acc, roc, pr = tr.evaluate({"movieId": t["movieId"], "userId": t["userId"], "label": t["label"]})
        assert tr.iterations == 5 * 7403
    assert sorted(hist) == ["accuracy", "auc", "auc_1", "loss"] and all(len(v) == 5 for v in hist.values())
    got = {"loss": loss, "accuracy": acc, "roc_auc": roc, "pr_auc": pr}
    print("two towers end to end:", got, "loss per epoch", hist["loss"])
    for k, (lo, hi) in _band(fit).items():
        assert lo <= got[k] <= hi, (k, got[k], (lo, hi))
    oracle0 = fit["runs"][0]["history"]
    # the training history follows the oracle's seed-0 run closely in the first epoch
    assert abs(hist["loss"][0] - oracle0[0]["loss"]) < 5e-3
    assert abs(hist["auc"][0] - oracle0[0]["roc_auc"]) < 5e-3
