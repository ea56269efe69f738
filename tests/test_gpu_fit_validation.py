"""GPU checks of validation during `fit` and of `Trainer.evaluate` (csrc/trainer.cu, DESIGN.md section 4.10):
validation is `evaluate` of the epoch's weights and changes nothing else, agrees with the float64 oracle's validated
fit (oracle/fit_validation.py), and follows Keras's validation_split / validation_freq rules."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import fit_validation, keras_eval, ncf_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CUDACORE = {"deepfm_impl": "cudacore"}       # the kernel the trainer's forward shares its bits with
SPREAD_MULTIPLE = 4.0                        # as tests/test_gpu_fit.py: GPU-to-float64 in float32-to-float64 units
MODELS = ["neuralcf", "deepfm"]


@pytest.fixture(scope="module")
def data():
    out = {}
    for m in MODELS:
        z = dict(np.load(os.path.join(GOLDEN, "%s_trainset.npz" % m)))
        out[m] = {k: v for k, v in z.items() if m == "deepfm" or k in ("movieId", "userId", "label")}
    t = dict(np.load(os.path.join(GOLDEN, "neuralcf_002_testset.npz")))
    out["neuralcf_test"] = {k: t[k] for k in ("movieId", "userId", "label")}
    out["deepfm_test"] = dict(np.load(os.path.join(GOLDEN, "dien_testset.npz")))
    return out


def _split(data, model, n, nv):
    """n training rows and nv validation rows (the model's test set, spread over it)."""
    f = {k: np.ascontiguousarray(v[:n]) for k, v in data[model].items()}
    test = data[model + "_test"]
    idx = np.linspace(0, len(test["label"]) - 1, nv).astype(np.int64)
    return f, {k: np.ascontiguousarray(v[idx]) for k, v in test.items()}


def _same_weights(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def _counts_and_bits(r, s):
    assert (r.rows, r.positives, r.correct) == (s.rows, s.positives, s.correct)
    assert (r.loss, r.accuracy, r.roc_auc, r.pr_auc) == (s.loss, s.accuracy, s.roc_auc, s.pr_auc)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [12, 33])
@pytest.mark.parametrize("model", MODELS)
def test_validation_is_evaluate_of_the_epochs_weights(data, model, B):
    """val_history[e] is CTRModel.evaluate (CUDA cores, one batch) of the weights after epoch e, counts exact and
    metrics bit for bit; those weights come from a second trainer advanced one epoch per fit, whose fits together
    give the 3-epoch fit's bits (weights, iterations, history); its Trainer.evaluate is the same result."""
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec(model)
    W0 = init_weights(spec, 1, for_test=False)
    n, epochs = 3000, 3
    f, val = _split(data, model, n, 1000)
    orders = ncf_train.epoch_orders(n, epochs, 7)
    with Trainer(spec, W0) as tr:
        res, vres, validated = tr._fit(f, epochs=epochs, batch_size=B, order=orders, validation_data=val)
        W3, it3 = tr.weights(), tr.iterations
    assert validated == [0, 1, 2]
    with Trainer(spec, W0) as tr:
        for e in range(epochs):
            (r,), _, _ = tr._fit(f, epochs=1, batch_size=B, order=orders[e:e + 1])
            _counts_and_bits(r, res[e])
            with CTRModel(spec, tr.weights(), options=CUDACORE) as m:
                ref = m.evaluate_result(val)
            assert ref.rows == 1000
            _counts_and_bits(vres[e], ref)
            _counts_and_bits(tr.evaluate_result(val), ref)
            assert tr.evaluate(val) == (ref.loss, ref.accuracy, ref.roc_auc, ref.pr_auc)
        _same_weights(tr.weights(), W3)
        assert tr.iterations == it3 == epochs * -(-n // B)


@pytest.mark.gpu
@pytest.mark.parametrize("B,n,epochs", [(12, 2000, 2), (4096, 20000, 2)])
@pytest.mark.parametrize("model", MODELS)
def test_validation_changes_nothing_else(data, model, B, n, epochs):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec(model)
    W0 = init_weights(spec, 2, for_test=False)
    f, val = _split(data, model, n, 700)
    outs = []
    for v in (None, val):
        with Trainer(spec, W0) as tr:
            h = tr.fit(f, epochs=epochs, batch_size=B, seed=3, validation_data=v)
            outs.append((h, tr.weights(), tr.iterations))
    (h0, W_0, it0), (h1, W_1, it1) = outs
    assert sorted(h1) == sorted(list(h0) + ["val_loss", "val_accuracy", "val_auc", "val_auc_1"])
    assert {k: h1[k] for k in h0} == h0 and it0 == it1
    assert all(len(v) == epochs for v in h1.values())
    _same_weights(W_0, W_1)


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_validation_agrees_with_the_float64_oracle(data, model):
    """Loss: within 4x the float32 oracle's own distance from float64 (plus 4 float32 ulps of the loss).  Accuracy
    and AUCs: a row's counts move only when a threshold lies between its GPU and its float64 probability; with
    `cross` such (row, threshold) pairs, the 0.5 crossings bound the accuracy by crossings / rows, and each
    crossing moves one count of one threshold, which moves the ROC AUC by at most 1 / min(P, N) (its two
    trapezoids) and the interpolated PR AUC by at most 3 / min(P, N) (two segments' recall widths and one
    precision).  The GPU probabilities are those of the CUDA-core model of each epoch's weights, which
    validation reports bit for bit (test_validation_is_evaluate_of_the_epochs_weights)."""
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec(model)
    W0 = init_weights(spec, 5, for_test=False)
    n, B, epochs = 2000, 33, 3
    f, val = _split(data, model, n, 1000)
    orders = ncf_train.epoch_orders(n, epochs, 9)
    _, _, v64, _ = fit_validation.fit(model, W0, f, orders, B, np.float64, val=val)
    _, _, v32, _ = fit_validation.fit(model, W0, f, orders, B, np.float32, val=val)
    thresholds = np.asarray(keras_eval.keras_thresholds(), np.float32)
    y = np.asarray(val["label"])
    P, N = int(y.sum()), int(len(y) - y.sum())
    W64 = ncf_train.as_dtype(W0, np.float64)
    opt64 = None
    with Trainer(spec, W0) as tr:
        for e in range(epochs):
            h = tr.fit(f, epochs=1, batch_size=B, order=orders[e:e + 1], validation_data=val)
            W64, _, _, opt64 = fit_validation.fit(model, W64, f, orders[e:e + 1], B, np.float64, opt=opt64)
            with CTRModel(spec, tr.weights(), options=CUDACORE) as m:
                pg = m.predict(val)[:, 0]
            p64 = _forward(model, W64, val).astype(np.float32)      # keras_evaluate counts float32(p)
            spread = abs(v32[e]["loss"] - v64[e]["loss"])
            err = abs(h["val_loss"][0] - v64[e]["loss"])
            assert err <= SPREAD_MULTIPLE * spread + 4 * np.spacing(np.float32(v64[e]["loss"])), (e, err, spread)
            # p > t differs between the two exactly when lo <= t < hi
            lo, hi = np.minimum(pg, p64), np.maximum(pg, p64)
            cross = int(((thresholds[None, :] >= lo[:, None]) & (thresholds[None, :] < hi[:, None])).sum())
            half = int(((np.float32(0.5) >= lo) & (np.float32(0.5) < hi)).sum())
            print(model, "epoch", e, "loss err / spread", err, spread, "crossings", cross, "at 0.5", half)
            assert abs(h["val_accuracy"][0] - v64[e]["accuracy"]) <= half / len(y) + 1e-12
            assert abs(h["val_auc"][0] - v64[e]["roc_auc"]) <= cross / min(P, N) + 1e-12
            assert abs(h["val_auc_1"][0] - v64[e]["pr_auc"]) <= 3 * cross / min(P, N) + 1e-12


def _forward(model, W, val):
    from oracle import deepfm_train
    if model == "neuralcf":
        return ncf_train.forward(W, val["movieId"], val["userId"], np.float64)[0]
    return deepfm_train.forward(W, deepfm_train.Rows.from_features(val), np.float64)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_validation_split_is_validation_data_of_the_last_rows(data, model):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec(model)
    W0 = init_weights(spec, 6, for_test=False)
    f = {k: np.ascontiguousarray(v[:403]) for k, v in data[model].items()}
    at = 302                                                   # floor(403 * 0.75)
    outs = []
    with Trainer(spec, W0) as tr:
        outs.append((tr.fit(f, epochs=2, batch_size=12, seed=4, validation_split=0.25), tr.weights()))
    with Trainer(spec, W0) as tr:
        head = {k: v[:at] for k, v in f.items()}
        tail = {k: v[at:] for k, v in f.items()}
        outs.append((tr.fit(head, epochs=2, batch_size=12, seed=4, validation_data=tail), tr.weights()))
        assert tr.iterations == 2 * -(-at // 12)
    assert outs[0][0] == outs[1][0] and len(outs[0][0]["val_loss"]) == 2
    _same_weights(outs[0][1], outs[1][1])


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_validation_freq_logs_only_the_validated_epochs(data, model):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec(model)
    W0 = init_weights(spec, 7, for_test=False)
    f, val = _split(data, model, 500, 300)
    hs = []
    for freq in (1, 2):
        with Trainer(spec, W0) as tr:
            hs.append(tr.fit(f, epochs=5, batch_size=33, seed=2, validation_data=(val, val["label"]),
                             validation_freq=freq))
    every, second = hs
    for k in ("loss", "accuracy", "auc", "auc_1"):
        assert every[k] == second[k]
        assert len(every["val_" + k]) == 5 and len(second["val_" + k]) == 2
        assert second["val_" + k] == [every["val_" + k][1], every["val_" + k][3]]


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_validated_fit_is_deterministic(data, model):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec(model)
    W0 = init_weights(spec, 8, for_test=False)
    f, val = _split(data, model, 3000, 1000)
    outs = []
    for _ in range(2):
        with Trainer(spec, W0) as tr:
            outs.append((tr.fit(f, epochs=2, batch_size=33, seed=5, validation_data=val), tr.weights()))
    assert outs[0][0] == outs[1][0]
    _same_weights(outs[0][1], outs[1][1])


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_rejected_validation_leaves_the_trainer_unchanged(data, model):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec(model)
    f, val = _split(data, model, 100, 60)
    at = np.arange(60)
    bad = [(ValueError, "label", dict(val, label=np.where(at == 50, 2, val["label"]).astype(np.int32))),
           (ValueError, "movieId", dict(val, movieId=np.where(at == 59, 1001, val["movieId"]).astype(np.int32))),
           (ValueError, "userId", dict(val, userId=np.where(at == 0, -1, val["userId"]).astype(np.int32)))]
    if model == "deepfm":
        bad += [(ValueError, "genre", dict(val, movieGenre1=np.where(at == 40, 19, val["movieGenre1"]).astype(np.int32))),
                (KeyError, "userRatingStddev", {k: v for k, v in val.items() if k != "userRatingStddev"})]
    with Trainer(spec, init_weights(spec, 9, for_test=False)) as tr:
        tr.fit(f, epochs=1, batch_size=12, seed=0)
        before, it = tr.weights(), tr.iterations
        for exc, what, v in bad:
            with pytest.raises(exc, match=what):
                tr.fit(f, epochs=1, validation_data=v)
            with pytest.raises(exc, match=what):
                tr.evaluate(v)
        assert tr.iterations == it
        _same_weights(before, tr.weights())
        h = tr.fit(f, epochs=1, batch_size=12, seed=0, validation_data=val)       # and it still trains
        assert tr.iterations == it + 9 and len(h["val_loss"]) == 1


_FRESH_EVALUATE = """
import json, os, sys
import numpy as np
from sparrowrecsys_b200.model import CTRModel
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.training import Trainer
from sparrowrecsys_b200.weights import init_weights
test = dict(np.load(os.path.join(sys.argv[1], "dien_testset.npz")))
val = {k: np.ascontiguousarray(v[:500]) for k, v in test.items()}
spec = default_spec("deepfm", emb_dim=64)
with Trainer(spec, init_weights(spec, 3, for_test=True)) as tr:
    got = tr.evaluate(val)
    W = tr.weights()
with CTRModel(spec, W, options={"deepfm_impl": "cudacore"}) as m:
    ref = m.evaluate(val, batch_size=500)
print(json.dumps([list(got), list(ref)]))
"""


@pytest.mark.gpu
def test_deepfm_trainer_evaluates_in_a_process_without_a_model():
    """The trainer's DeepFM forward is deepfm_kernel, whose dynamic shared memory opt-in (at E = 64, above the 48 KiB
    default) srs_model_create also sets: a trainer created in a fresh process, before any CTRModel, must set it itself.
    Its evaluate then equals that of a model rebuilt from its weights."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _FRESH_EVALUATE, GOLDEN], capture_output=True, text=True, cwd=root,
                       timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    got, ref = json.loads(r.stdout.strip().splitlines()[-1])
    assert got == ref


@pytest.mark.gpu
def test_abi_rejects_bad_validation_rows_before_any_launch(data):
    """The library's own checks past encode_batch: a validation genre >= n_genres is SRS_ERR_RANGE naming the
    validation data, a missing validation column or val_freq < 1 SRS_ERR_INVALID; the trainer is unchanged."""
    from sparrowrecsys_b200 import _lib
    from sparrowrecsys_b200.features import encode_batch
    from sparrowrecsys_b200.model import _host_struct
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("deepfm")
    f, val = _split(data, "deepfm", 50, 30)
    with Trainer(spec, init_weights(spec, 10, for_test=False)) as tr:
        before = tr.weights()
        keep = []
        b = _host_struct(encode_batch(spec, f), keep)
        lab = np.ascontiguousarray(f["label"], np.int32)
        vlab = np.ascontiguousarray(val["label"], np.int32)
        order = np.arange(50, dtype=np.int32)

        def call(vb, freq=1):
            return tr._lib.srs_trainer_fit_validate_host(tr._h, C.byref(b), lab.ctypes.data, order.ctypes.data, 12, 1,
                                                         None, C.byref(vb), vlab.ctypes.data, freq, None)
        enc = encode_batch(spec, val)
        enc.user_genre[7, 0] = 19
        rc = call(_host_struct(enc, keep))
        assert rc == _lib.SRS_ERR_RANGE and b"validation data: userGenre1" in tr._lib.srs_last_error()
        vb = _host_struct(encode_batch(spec, val), keep)
        vb.numerics = None
        assert call(vb) == _lib.SRS_ERR_INVALID
        assert tr._lib.srs_trainer_evaluate_host(tr._h, C.byref(vb), vlab.ctypes.data,
                                                 C.byref(_lib.SrsEvalResult())) == _lib.SRS_ERR_INVALID
        assert call(_host_struct(encode_batch(spec, val), keep), freq=0) == _lib.SRS_ERR_INVALID
        assert tr.iterations == 0
        _same_weights(before, tr.weights())


def _band(fit):
    """The seed band of the oracle's test metrics, widened by half its width on each side (tests/test_gpu_fit.py)."""
    return {k: (lo - (hi - lo) / 2, hi + (hi - lo) / 2) for k, (lo, hi) in fit["band"].items()}


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_the_script_end_to_end_with_validation(data, model):
    """load(seed=0), fit(train, epochs=5, validation_data=test) at batch 12: the last val_* entries are
    evaluate(test) after the fit (one batch), inside the oracle's band."""
    import tfrecmodel
    mod = getattr(tfrecmodel, model)
    with open(os.path.join(GOLDEN, "%s_fit.json" % model)) as fh:
        band = _band(json.load(fh))
    test = data[model + "_test"]
    mod.load(seed=0)
    hist = mod.fit(data[model], epochs=5, batch_size=12, seed=0, validation_data=test)
    assert all(len(v) == 5 for v in hist.values()) and len(hist) == 8
    loss, acc, roc, pr = mod.evaluate(test)
    assert (hist["val_loss"][-1], hist["val_accuracy"][-1], hist["val_auc"][-1], hist["val_auc_1"][-1]) == \
        (loss, acc, roc, pr)
    got = {"loss": loss, "accuracy": acc, "roc_auc": roc, "pr_auc": pr}
    print(model, "end to end with validation:", got, "val_loss per epoch", hist["val_loss"])
    for k, (lo, hi) in band.items():
        assert lo <= got[k] <= hi, (k, got[k], band[k])


def test_the_surfaces_take_the_validation_keywords_and_the_others_still_do_not_fit():
    import inspect
    from tfrecmodel import deepfm, din, neuralcf, twotowers
    for mod in (neuralcf, deepfm):
        params = inspect.signature(mod.fit).parameters
        assert {"validation_data", "validation_split", "validation_freq"} <= set(params)
    for mod in (din, twotowers):
        with pytest.raises(NotImplementedError, match="NeuralCF"):
            mod.fit({"movieId": np.zeros(1, np.int32)})
