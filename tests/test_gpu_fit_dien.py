"""GPU checks of DIEN's `fit` (csrc/dien_train.cu and srs_trainer_fit_dien_host in csrc/trainer.cu, DESIGN.md
section 4.20) against the float64 / float32 oracle (oracle/dien_train.py)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import ctr_oracle, dien_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_aux_weights, init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SPREAD_MULTIPLE = 4.0          # GPU-to-float64 distance allowed, in units of the float32-to-float64 distance
# the batch-4096 case at EP = 32 needs more (DESIGN.md section 4.20): after one step the AUGRU's gate kernels sit in
# Adam's epsilon regime, where a gradient's last bits decide the update; on an NVIDIA H100 80GB HBM3 at 700 W
# augru_z_input/kernel measured 6.4x the float32 spread at batch 4096
CASE_MULTIPLE = {(32, 5, 4096, 4096): 7.0}


def _weights(spec, seed):
    W = {**init_weights(spec, seed), **init_aux_weights(spec, seed)}
    rng = np.random.default_rng(seed + 50)
    for k in W:                # non-zero biases and PReLU alphas, so every tensor shows in the outputs
        if k.endswith("/bias") or k.endswith("/alpha"):
            W[k] = rng.uniform(-0.3, 0.3, size=W[k].shape).astype(np.float32)
    return W


def _features(spec, n, seed):
    """n synthetic rows with negatives and labels; padded history slots at the start, middle and end of rows, one
    all-padding history, a candidate equal to a history id, missing genres."""
    from sparrowrecsys_b200.features import negative_history, synthetic_features
    from oracle.ctr_oracle import din_history_keys
    f = synthetic_features(spec, n, seed=seed)
    keys = din_history_keys(spec.hist_len)
    for k in keys:
        f[k] = np.array(f[k])
    rng = np.random.default_rng(seed)
    for i in range(n):
        if i % 4 == 1:
            f[keys[0]][i] = 0
        if i % 4 == 2:
            f[keys[len(keys) // 2]][i] = 0
        if i % 4 == 3:
            f[keys[-1]][i] = 0
    if n > 5:
        for k in keys:
            f[k][5] = 0
        f["movieId"] = np.array(f["movieId"])
        f["movieId"][4] = f[keys[0]][4]
    for g in ("movieGenre1", "userGenre1"):
        f[g] = np.array(f[g], dtype=object)
        f[g][::7] = ""
    f.update(negative_history(f, spec.hist_len, seed, n_movies=spec.n_movies))
    f["label"] = (rng.random(n) < 0.4).astype(np.int32)
    return f


def _check_close(got, w64, w32, what):
    m = CASE_MULTIPLE.get(what, SPREAD_MULTIPLE)
    worst = 0.0
    for k in w64:
        d_gpu = np.abs(got[k].astype(np.float64) - w64[k]).max()
        d_32 = np.abs(w32[k].astype(np.float64) - w64[k]).max()
        ulp = np.spacing(np.float32(np.abs(w64[k]).max()))
        worst = max(worst, (d_gpu - ulp) / d_32 if d_32 > 0 else 0.0)
        assert d_gpu <= m * d_32 + ulp, (what, k, d_gpu, d_32)
    print("worst spread ratio", what, worst)


# (E, T, hidden, n_movies, batch, rows, epochs): long horizons and large batches at the reference shape, 100 steps
# of one row, 100 of 12 and 33 rows, one and ten of 4096; tests/test_fit_matrix.py holds every EP, hidden width,
# history length and padding edge to the same rule
MATRIX = [(12, 5, (128, 64), 3000, 1, 100, 1), (10, 5, (128, 64), 3000, 12, 1200, 1),
          (16, 5, (128, 64), 3000, 33, 3300, 1), (10, 5, (128, 64), 3000, 4096, 40960, 1),
          (32, 5, (128, 64), 3000, 4096, 4096, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("E,T,hidden,n_movies,B,n,epochs", MATRIX)
def test_fit_matches_the_float64_oracle(E, T, hidden, n_movies, B, n, epochs):
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("dien", emb_dim=E, hist_len=T, hidden=hidden, n_movies=n_movies, n_users=500)
    W = _weights(spec, E + T)
    f = _features(spec, n, seed=n + E)
    rows = dien_train.Rows.from_features(f, T)
    orders = [np.arange(n)] * epochs
    w64, h64, _ = dien_train.fit(W, rows, orders, B, np.float64)
    w32, h32, _ = dien_train.fit(W, rows, orders, B, np.float32)
    with Trainer(spec, W) as tr:
        hist = tr.fit(f, epochs=epochs, batch_size=B)
        got = tr.weights()
    assert np.array_equal(got["augru_h0"], W["augru_h0"])
    _check_close(got, w64, w32, (E, T, B, n))
    for e in range(epochs):                 # the history is held to the same rule, plus a float32 rounding
        for k in ("loss", "auc", "auc_value"):
            spread = abs(h32[e][k] - h64[e][k])
            assert abs(hist[k][e] - h64[e][k]) <= SPREAD_MULTIPLE * spread + 1e-6, (k, e, hist[k][e], h64[e][k], spread)


@pytest.mark.gpu
def test_one_step_reports_dien_evaluate_and_a_second_fit_gives_the_same_bits():
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("dien", n_movies=3000, n_users=500)
    W = _weights(spec, 3)
    f = _features(spec, 100, seed=3)
    with CTRModel(spec, W) as m:
        want = m.dien_evaluate(f)                        # one batch
    runs = []
    for _ in range(2):
        with Trainer(spec, W) as tr:
            h = tr.fit(f, epochs=1, batch_size=100)
            assert tr.iterations == 1
            runs.append((h, tr.weights()))
    assert runs[0][0] == {k: [v] for k, v in want.items()}
    assert runs[0][0] == runs[1][0]
    assert all(np.array_equal(runs[0][1][k], runs[1][1][k]) for k in W)
    assert np.array_equal(runs[0][1]["augru_h0"], W["augru_h0"])


@pytest.mark.gpu
def test_rejected_calls_change_nothing_and_the_trained_model_serves_what_the_oracle_predicts():
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("dien", emb_dim=16, n_movies=3000, n_users=500)
    W = _weights(spec, 5)
    f = _features(spec, 60, seed=5)
    with Trainer(spec, W) as tr:
        with pytest.raises(ValueError):
            tr.fit(f, epochs=1, batch_size=12, order=np.zeros((1, 60), np.int32))
        bad = dict(f, negtive_userRatedMovie3=np.full(60, spec.n_movies))
        with pytest.raises(ValueError):
            tr.fit(bad, epochs=1, batch_size=12)
        with pytest.raises(KeyError):
            tr.fit({k: v for k, v in f.items() if k != "negtive_userRatedMovie5"}, epochs=1)
        with pytest.raises(NotImplementedError):
            tr.fit(f, validation_split=0.5)
        with pytest.raises(NotImplementedError, match="dien_evaluate"):
            tr.evaluate(f)
        assert tr.iterations == 0
        now = tr.weights()
        assert all(np.array_equal(now[k], W[k]) for k in W)
        order = np.stack([np.random.default_rng(1).permutation(60)])
        tr.fit(f, epochs=1, batch_size=12, order=order)
        trained = tr.weights()
        with tr.to_model() as m:
            p = m.predict(f)
    w64, _, _ = dien_train.fit(W, dien_train.Rows.from_features(f, 5), order, 12, np.float64)
    p64, _ = ctr_oracle.dien_forward(spec, w64, f, np.float64)
    p_tr, _ = ctr_oracle.dien_forward(spec, trained, f, np.float64)
    assert np.abs(p - p_tr).max() <= 1e-5
    assert np.abs(p - p64).max() <= 1e-4


@pytest.mark.gpu
def test_tfrecmodel_fit_trains_in_file_order():
    import tfrecmodel.dien as D
    spec = default_spec("dien", n_movies=1001)
    f = _features(spec, 48, seed=9)
    D.load(seed=2)
    w0 = dict(D._surface.weights)
    h = D.fit(f, epochs=2, batch_size=12)
    assert set(h) == {"loss", "auc", "auc_value"} and len(h["loss"]) == 2
    rows = dien_train.Rows.from_features(f, 5)
    _, h64, _ = dien_train.fit(w0, rows, [np.arange(48)] * 2, 12, np.float64)
    _, h32, _ = dien_train.fit(w0, rows, [np.arange(48)] * 2, 12, np.float32)
    for e in range(2):
        assert abs(h["loss"][e] - h64[e]["loss"]) <= SPREAD_MULTIPLE * abs(h32[e]["loss"] - h64[e]["loss"]) + 1e-6
    assert np.array_equal(D._surface.weights["augru_h0"], w0["augru_h0"])


@pytest.mark.gpu
def test_the_other_entry_points_reject_a_dien_trainer_and_ids_are_checked_before_any_launch():
    from sparrowrecsys_b200 import _lib
    from sparrowrecsys_b200.training import Trainer
    spec = default_spec("dien", n_movies=3000, n_users=500)
    W = _weights(spec, 6)
    f = _features(spec, 24, seed=6)
    with Trainer(spec, W) as tr:
        lib = tr._lib
        keep = []
        batch, lab, n = tr._rows(f, None, keep, "fit")
        order = np.arange(n, dtype=np.int32)
        res = (_lib.SrsEvalResult * 1)()
        for rc in (lib.srs_trainer_fit_host(tr._h, C.byref(batch), lab.ctypes.data, order.ctypes.data, 12, 1, res),
                   lib.srs_trainer_fit_validate_host(tr._h, C.byref(batch), lab.ctypes.data, order.ctypes.data, 12, 1,
                                                     res, None, None, 1, None),
                   lib.srs_trainer_evaluate_host(tr._h, C.byref(batch), lab.ctypes.data, res)):
            assert rc == _lib.SRS_ERR_INVALID and b"srs_trainer_fit_dien_host" in lib.srs_last_error()
        # an id no float32 holds near the int32 limit, at the ABI (the Python layer range-checks before it)
        neg = np.ascontiguousarray(np.stack([f["negtive_userRatedMovie%d" % k] for k in range(2, 6)], 1), np.int32)
        hist = C.cast(batch.hist, C.POINTER(C.c_int32))
        saved = hist[7 * batch.hist_stride + 2]
        for bad in (2 ** 31 - 1, -2 ** 31, spec.n_movies):
            hist[7 * batch.hist_stride + 2] = bad
            rc = lib.srs_trainer_fit_dien_host(tr._h, C.byref(batch), neg.ctypes.data, 4, lab.ctypes.data,
                                               order.ctypes.data, 12, 1, None)
            assert rc == _lib.SRS_ERR_RANGE and b"history id" in lib.srs_last_error(), bad
        hist[7 * batch.hist_stride + 2] = saved
        assert tr.iterations == 0
        now = tr.weights()
        assert all(np.array_equal(now[k], W[k]) for k in W)


def _script_rows(part):
    """DIEN.py's rows with their negatives (:49-50), from the committed fixtures (make_dien_train_golden.py)."""
    from sparrowrecsys_b200.features import negative_history
    if part == "train":
        z = dict(np.load(os.path.join(GOLDEN, "deepfm_trainset.npz")))
        z["userRatedMovie1"] = np.load(os.path.join(GOLDEN, "widendeep_samples.npz"))["train_userRatedMovie1"]
        z.update(dict(np.load(os.path.join(GOLDEN, "dien_train_samples.npz"))))
        seed = 2020
    else:
        z = dict(np.load(os.path.join(GOLDEN, "dien_testset.npz")))
        seed = 2021
    z.update(negative_history(z, 5, seed))
    return z


@pytest.mark.gpu
def test_the_script_end_to_end():
    """DIEN.py: an untrained model, fit(train, epochs=5) at batch 12 in file order, then evaluate on testSamples at
    batch 12; the test metrics land inside the float32 oracle's seed-to-seed band, widened by half its width on
    each side (as the other models' end-to-end checks)."""
    import tfrecmodel.dien as D
    with open(os.path.join(GOLDEN, "dien_fit.json")) as fh:
        fit = json.load(fh)
    train, test = _script_rows("train"), _script_rows("test")
    assert len(train["label"]) == fit["rows"] == 88827 and len(test["label"]) == fit["test_rows"]
    D.load(seed=0)
    hist = D.fit(train, epochs=fit["epochs"], batch_size=fit["batch_size"])
    assert len(hist["loss"]) == 5
    got = D.evaluate_outputs(test, batch_size=fit["batch_size"])
    band = {k: (lo - (hi - lo) / 2, hi + (hi - lo) / 2) for k, (lo, hi) in fit["band"].items()}
    print("dien end to end:", got, "history", hist, "band", fit["band"])
    for k, (lo, hi) in band.items():
        assert lo <= got[k] <= hi, (k, got[k], band[k])
    # the oracle run of the same seed trained the same rows in the same order
    run0 = fit["runs"][0]
    assert run0["seed"] == 0 and run0["iterations"] == 5 * -(-88827 // 12)
