"""GPU checks of NeuralCF's `fit` (csrc/ncf_train.cu, csrc/trainer.cu, DESIGN.md section 4.8) against the float64 / float32 oracle
(oracle/ncf_train.py) and the reference script's end-to-end known answer (tests/golden/neuralcf_fit.json)."""
import json
import os
import threading

import numpy as np
import pytest

from oracle import keras_eval, ncf_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SPREAD_MULTIPLE = 4.0          # GPU-to-float64 distance allowed, in units of the float32-to-float64 distance


@pytest.fixture(scope="module")
def trainset():
    z = np.load(os.path.join(GOLDEN, "neuralcf_trainset.npz"))
    return {k: z[k] for k in ("movieId", "userId", "label")}


def _rows(ts, n, one_movie=False):
    f = {k: np.ascontiguousarray(v[:n]) for k, v in ts.items()}
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


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,epochs", CASES)
def test_short_horizon_parity(trainset, B, n, epochs):
    assert _steps(B, n, epochs) in (1, 2, 10, 100)
    _parity(trainset, B, n, epochs, one_movie=False)


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,epochs", [(33, 66, 1), (12, 40, 3)])
def test_parity_batch_of_one_movie(trainset, B, n, epochs):
    _parity(trainset, B, n, epochs, one_movie=True)


def _parity(trainset, B, n, epochs, one_movie):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("neuralcf")
    W0 = init_weights(spec, 3, for_test=True)
    f = _rows(trainset, n, one_movie)
    orders = ncf_train.epoch_orders(n, epochs, 11)
    args = (W0, f["movieId"], f["userId"], f["label"], orders, B)
    W64, _, _, _ = ncf_train.fit(*args, dtype=np.float64)
    W32, _, _, _ = ncf_train.fit(*args, dtype=np.float32)
    with Trainer(spec, W0) as tr:
        tr.fit(f, epochs=epochs, batch_size=B, order=orders)
        assert tr.iterations == _steps(B, n, epochs)
        Wg = tr.weights()
    for k in W0:
        spread = float(np.abs(W32[k] - W64[k]).max())
        err = float(np.abs(Wg[k].astype(np.float64) - W64[k]).max())
        moved = float(np.abs(W64[k] - W0[k]).max())
        assert moved > 0, k
        assert err <= SPREAD_MULTIPLE * spread + 1e-9, (k, err, spread)


@pytest.mark.gpu
def test_fit_is_deterministic(trainset):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("neuralcf")
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
def test_history_matches_keras_evaluate_of_the_oracle_steps(trainset):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("neuralcf")
    W0 = init_weights(spec, 5, for_test=False)
    n, B, epochs = 600, 12, 2
    f = _rows(trainset, n)
    orders = ncf_train.epoch_orders(n, epochs, 2)
    _, _, out, _ = ncf_train.fit(W0, f["movieId"], f["userId"], f["label"], orders, B, np.float64, keep_outputs=True)
    with Trainer(spec, W0) as tr:
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


def _band(fit):
    """The seed-to-seed band of the oracle's test metrics, widened by half its width on each side: the GPU run starts
    from seed 0's weights and order but its rounding parts ways over 37 015 steps, so it is one more draw."""
    out = {}
    for k, (lo, hi) in fit["band"].items():
        w = hi - lo
        out[k] = (lo - w / 2, hi + w / 2)
    return out


@pytest.mark.gpu
def test_the_script_end_to_end(trainset):
    """NeuralCF.py:74-91: an untrained model, fit(train, epochs=5) at batch 12, then evaluate on testSamples."""
    from tfrecmodel import neuralcf
    with open(os.path.join(GOLDEN, "neuralcf_fit.json")) as fh:
        fit = json.load(fh)
    neuralcf.load(seed=0)
    hist = neuralcf.fit(trainset, epochs=5, batch_size=12, seed=0)
    assert sorted(hist) == ["accuracy", "auc", "auc_1", "loss"] and all(len(v) == 5 for v in hist.values())
    z = np.load(os.path.join(GOLDEN, "neuralcf_002_testset.npz"))
    test = {"movieId": z["movieId"], "userId": z["userId"], "label": z["label"]}
    loss, acc, roc, pr = neuralcf.evaluate(test, batch_size=12)
    band = _band(fit)
    got = {"loss": loss, "accuracy": acc, "roc_auc": roc, "pr_auc": pr}
    for k, (lo, hi) in band.items():
        assert lo <= got[k] <= hi, (k, got[k], band[k])
    oracle0 = fit["runs"][0]["history"]
    # the training history follows the oracle's seed-0 run closely in the first epoch
    assert abs(hist["loss"][0] - oracle0[0]["loss"]) < 5e-3
    assert abs(hist["auc"][0] - oracle0[0]["roc_auc"]) < 5e-3
    p = neuralcf.predict({"movieId": test["movieId"][:4], "userId": test["userId"][:4]})
    assert p.shape == (4, 1)


@pytest.mark.gpu
def test_trained_model_serves(trainset):
    from sparrowrecsys_b200 import serving
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("neuralcf")
    with Trainer(spec, init_weights(spec, 6, for_test=False)) as tr:
        tr.fit(_rows(trainset, 2000), epochs=1, batch_size=12, seed=1)
        W = tr.weights()
        m = tr.to_model()
    f = {"movieId": trainset["movieId"][-300:], "userId": trainset["userId"][-300:]}
    p = m.predict(f)
    po, _, _ = ncf_train.forward(W, f["movieId"], f["userId"], np.float64)
    assert np.abs(p[:, 0] - po).max() <= 2e-6
    srv = serving.serve({"recmodel": (spec, m.predict)}, "127.0.0.1", 0)
    th = threading.Thread(target=srv.serve_forever, daemon=True)
    th.start()
    try:
        import urllib.request
        body = json.dumps({"instances": [{"movieId": int(f["movieId"][i]), "userId": int(f["userId"][i])}
                                         for i in range(3)]}).encode()
        req = urllib.request.Request("http://127.0.0.1:%d/v1/models/recmodel:predict" % srv.server_address[1],
                                     data=body, headers={"Content-Type": "application/json"})
        out = json.loads(urllib.request.urlopen(req, timeout=60).read())
        np.testing.assert_allclose(np.array(out["predictions"])[:, 0], p[:3, 0], rtol=0, atol=1e-6)
    finally:
        srv.shutdown()
        srv.server_close()
        th.join(timeout=10)
    m.close()


@pytest.mark.gpu
def test_rejected_fit_leaves_the_trainer_unchanged(trainset):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("neuralcf")
    f = _rows(trainset, 100)
    with Trainer(spec, init_weights(spec, 7, for_test=False)) as tr:
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
        assert tr.iterations == it
        after = tr.weights()
        assert all(np.array_equal(before[k], after[k]) for k in before)
        tr.fit(f, epochs=1, batch_size=12, seed=0)                  # and it still trains
        assert tr.iterations == it + 9


def test_other_models_do_not_fit():
    from tfrecmodel import din, twotowers
    for mod in (din, twotowers):
        with pytest.raises(NotImplementedError, match="NeuralCF"):
            mod.fit({"movieId": np.zeros(1, np.int32)})
