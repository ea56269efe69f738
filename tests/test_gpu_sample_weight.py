"""GPU checks of Keras's `sample_weight` / `class_weight` in `fit` and `evaluate` (DESIGN.md section 4.28): the
weighted step of every model against the float64 oracle at every step instantiation of the fit matrices, the bit
identities the weights must keep (no weights, all-ones weights, repeats, the step's forward, validation), weighted
`CTRModel.evaluate` of every evaluable kind and kernel against duplicated rows, and the rejections."""
import ctypes as C

import numpy as np
import pytest

import weighted_oracle as WO
from oracle import ncf_train, twotowers_train
from sparrowrecsys_b200.spec import default_spec
from test_evaluate import _cases, _labelled, _model
from test_fit_matrix import FIT_MATRIX, SERVING, FitCase, _case_id, _inputs, _rows, _spec
from test_fit_matrix import ORACLE as FIT_ORACLE
from test_fit_oracle_twotowers import TT_MATRIX, TTCase, case_id, case_spec, inputs
from test_sample_weight_oracle import row_weights

MODELS = ("neuralcf", "twotowers", "deepfm", "widendeep", "deepfm_v2")
CLASS_ONLY = {0: 0.25, 1: 3.0}


def _is_tt(c):
    return isinstance(c, TTCase)


def _cid(c):
    return "twotowers-" + case_id(c) if _is_tt(c) else _case_id(c)


def _c_spec(c):
    return case_spec(c) if _is_tt(c) else _spec(c)


def _c_inputs(c):
    return inputs(c) if _is_tt(c) else _inputs(c)


def _trainer(c, W):
    from sparrowrecsys_b200.training import Trainer
    return Trainer(_c_spec(c), W, adam=c.adam)


def _weighting(c):
    """(sample_weight, class_weight) of a case: seeds divisible by 4 weight by class only."""
    n = c.n
    if c.seed % 4 == 0:
        return None, CLASS_ONLY
    return row_weights(n, c.seed), ({0: 1.5, 1: 0.5} if c.seed % 4 == 1 else None)


def _oracle_weights(c):
    from sparrowrecsys_b200.training import sample_weights
    sw, cw = _weighting(c)
    return sample_weights(_c_inputs(c)[1]["label"], sw, cw)


def _reversed(orders, B):
    """Each batch's rows in reverse: another order of every sum over a batch."""
    return np.stack([np.concatenate([o[i:i + B][::-1] for i in range(0, len(o), B)]) for o in orders])


def _oracle_fit(c, dtype, reverse=False):
    W0, f, orders = _c_inputs(c)
    if reverse:
        orders = _reversed(orders, c.B)
    w = _oracle_weights(c)
    model = "twotowers" if _is_tt(c) else c.model
    data = (f["movieId"], f["userId"]) if model in ("neuralcf", "twotowers") else _rows(c)
    return WO.fit(model, W0, data, f["label"], orders, c.B, dtype, hp=c.adam, weights=w)[0]


def _check_parity(c, Wg):
    """The fit matrices' rule: within the case's multiple of the float32 oracle's distance from float64, plus one
    ulp of the tensor's largest value.  The distance is the larger of the float32 oracle's in the case's row order
    and with each batch's rows reversed: a weight of 1e3 among weights near 1 makes a batch's sums cancel, and one
    summation order of the float32 oracle can land by chance much nearer float64 than another (measured on an H100
    at 700 W: DeepFM_v2's proj_userId/bias after one weighted step of 4096 rows lands 7.1x the float32 spread in
    row order, 2.4x the spread with the rows reversed)."""
    W0 = _c_inputs(c)[0]
    W64, W32, W32r = _oracle_fit(c, np.float64), _oracle_fit(c, np.float32), _oracle_fit(c, np.float32, True)
    multiple = 4.0 if _is_tt(c) else c.multiple
    for k in W0:
        assert Wg[k].shape == W0[k].shape, k
        spread = max(float(np.abs(W32[k] - W64[k]).max()), float(np.abs(W32r[k] - W64[k]).max()))
        tol = multiple * spread + float(np.spacing(np.float32(np.abs(W64[k]).max())))
        err = float(np.abs(Wg[k].astype(np.float64) - W64[k]).max())
        assert err <= tol, (k, err, spread, tol)


def _fit(tr, c, f=None, **kw):
    W0, f0, orders = _c_inputs(c)
    sw, cw = _weighting(c)
    return tr.fit(f0 if f is None else f, epochs=c.epochs, batch_size=c.B, order=orders,
                  **dict(dict(sample_weight=sw, class_weight=cw), **kw))


# every EP (and NeuralCF / two-tower HP) of every changed step kernel: the fit matrices' cases without DIEN
MATRIX = [c for c in FIT_MATRIX if c.model != "dien"] + list(TT_MATRIX)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MATRIX, ids=_cid)
def test_weighted_fit_matches_float64_oracle(case):
    W0 = _c_inputs(case)[0]
    with _trainer(case, W0) as tr:
        _fit(tr, case)
        assert tr.iterations == case.epochs * -(-case.n // case.B)
        Wg = tr.weights()
    _check_parity(case, Wg)


def _horizon(model, B, n, epochs, seed):
    over = dict(n_movies=1000, n_users=1200)
    if model == "twotowers":
        return TTCase(dict(emb_dim=10, hidden=(10, 10), **over), B, n, epochs, seed, None)
    hidden = {"neuralcf": (10, 10), "deepfm": (64, 64), "widendeep": (128, 128), "deepfm_v2": (32, 16)}[model]
    return FitCase(model, dict(emb_dim=10, hidden=hidden, **over), B, n, epochs, seed, None)


# (B, n, epochs): 1, 2, 10 and 100 weighted steps; seed 4 weights by class only
HORIZON = [(1, 100, 1, 5), (12, 115, 1, 4), (12, 1190, 1, 6), (33, 50, 1, 6), (33, 320, 1, 5),
           (4096, 4096, 1, 7), (4096, 5000, 1, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("B,n,epochs,seed", HORIZON)
def test_short_horizon_weighted_parity(model, B, n, epochs, seed):
    c = _horizon(model, B, n, epochs, seed)
    assert epochs * -(-n // B) in (1, 2, 10, 100)
    with _trainer(c, _c_inputs(c)[0]) as tr:
        _fit(tr, c)
        Wg = tr.weights()
    _check_parity(c, Wg)


def _same(r, s):
    assert (r.rows, r.positives, r.correct) == (s.rows, s.positives, s.correct)
    assert (r.loss, r.accuracy, r.roc_auc, r.pr_auc) == (s.loss, s.accuracy, s.roc_auc, s.pr_auc)


def _same_weights(Wa, Wb):
    assert Wa.keys() == Wb.keys()
    for k in Wa:
        assert np.array_equal(Wa[k], Wb[k]), k


IDENTITY = {m: _horizon(m, 33, 320, 2, 5) for m in MODELS}


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_unit_weights_are_the_unweighted_fit_bit_for_bit(model):
    """No weights, all-ones sample weights and class_weight {0: 1, 1: 1} give the same weights and history, and
    launch the same number of kernels."""
    from sparrowrecsys_b200.model import launch_count
    c = IDENTITY[model]
    W0 = _c_inputs(c)[0]
    out = []
    for kw in (dict(sample_weight=None, class_weight=None), dict(sample_weight=np.ones(c.n, np.float32)),
               dict(class_weight={0: 1, 1: 1})):
        with _trainer(c, W0) as tr:
            n0 = launch_count()
            h = _fit(tr, c, **dict(dict(sample_weight=None, class_weight=None), **kw))
            launches = launch_count() - n0
            out.append((h, tr.weights(), launches))
    for h, W, launches in out[1:]:
        assert h == out[0][0]
        _same_weights(W, out[0][1])
        assert launches == out[0][2]


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_weighted_fit_repeats_and_matches_its_evaluate(model):
    """A second weighted fit has the same bits; a weighted fit launches as many kernels as an unweighted one; a
    one-step weighted history is weighted `Trainer.evaluate` of the starting weights, which is `to_model().evaluate`
    with the same weights."""
    from sparrowrecsys_b200.model import CTRModel, launch_count
    c = IDENTITY[model]
    W0, f, _ = _c_inputs(c)
    w = row_weights(c.n, 3)
    runs = []
    for _ in range(2):
        with _trainer(c, W0) as tr:
            n0 = launch_count()
            h = _fit(tr, c)
            runs.append((h, tr.weights(), launch_count() - n0))
    assert runs[0][0] == runs[1][0]
    _same_weights(runs[0][1], runs[1][1])
    with _trainer(c, W0) as tr:
        n0 = launch_count()
        _fit(tr, c, sample_weight=None, class_weight=None)
        assert launch_count() - n0 == runs[0][2]
    with _trainer(c, W0) as tr:
        r = tr.evaluate_result(f, sample_weight=w)
        h = tr.fit(f, epochs=1, batch_size=c.n, order=[np.arange(c.n)], sample_weight=w)
    assert (h["loss"][0], h["accuracy"][0], h["auc"][0], h["auc_1"][0]) == (r.loss, r.accuracy, r.roc_auc, r.pr_auc)
    name, options = SERVING.get(model, ("ncf_kernel<two_towers>", None))
    with CTRModel(_c_spec(c), W0, options=options) as m:
        assert m.kernel_name == name
        _same(m.evaluate_result(f, sample_weight=w), r)
    ref = WO.keras_evaluate(*_forward(c, W0, f), f["label"], w)
    assert abs(r.loss - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"]))


def _forward(c, W, f):
    """The float32 oracle's (p, z) of the rows."""
    if _is_tt(c):
        p, z, _ = twotowers_train.forward(W, f["movieId"], f["userId"], np.float32)
    elif c.model == "neuralcf":
        p, z, _ = ncf_train.forward(W, f["movieId"], f["userId"], np.float32)
    else:
        p, z, _ = FIT_ORACLE[c.model].forward(W, _rows(c), np.float32)
    return p, z


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_weighted_validation(model):
    """val_history[e] is weighted evaluate after epoch e (validation_data as (x, y, sample_weight), class_weight not
    applied to it), validation changes no weight and no training history, and validation_split splits the weights
    with the rows."""
    c = IDENTITY[model]
    W0, f, orders = _c_inputs(c)
    sw = row_weights(c.n, 8)
    cut = 250
    tr_f = {k: np.asarray(v)[:cut] for k, v in f.items()}
    va_f = {k: np.asarray(v)[cut:] for k, v in f.items()}
    tr_w, va_w = sw[:cut], sw[cut:]
    order = np.stack([np.random.default_rng(e).permutation(cut) for e in range(2)]).astype(np.int32)
    cw = {0: 0.5, 1: 2.0}
    with _trainer(c, W0) as tr:
        h = tr.fit(tr_f, epochs=2, batch_size=c.B, order=order, sample_weight=tr_w, class_weight=cw,
                   validation_data=(va_f, va_f["label"], va_w))
        Wv = tr.weights()
    with _trainer(c, W0) as tr:
        h0 = tr.fit(tr_f, epochs=2, batch_size=c.B, order=order, sample_weight=tr_w, class_weight=cw)
        _same_weights(tr.weights(), Wv)
    for k in h0:
        assert h[k] == h0[k], k
    with _trainer(c, W0) as tr:
        for e in range(2):
            tr.fit(tr_f, epochs=1, batch_size=c.B, order=order[e:e + 1], sample_weight=tr_w, class_weight=cw)
            r = tr.evaluate_result(va_f, sample_weight=va_w)
            assert (h["val_loss"][e], h["val_accuracy"][e], h["val_auc"][e], h["val_auc_1"][e]) == \
                (r.loss, r.accuracy, r.roc_auc, r.pr_auc)
    with _trainer(c, W0) as tr:
        hs = tr.fit(f, epochs=2, batch_size=c.B, order=order, sample_weight=sw, class_weight=cw,
                    validation_split=(c.n - cut) / c.n)
    assert hs == h


def _dup(f, k):
    return {key: np.repeat(np.asarray(v), k, axis=0) for key, v in f.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c[0] for c in _cases()])
def test_weighted_evaluate_is_duplicated_rows(case):
    """Integer weights: accuracy and both AUCs equal evaluate of each row repeated w times, bit for bit; the loss is
    sum w l / N; all-ones weights give the unweighted result; batches do not change the sums' bits."""
    name, spec, opts, kernel = [c for c in _cases() if c[0] == case][0]
    f = _labelled(spec, 700, 3)
    k = np.random.default_rng(5).integers(0, 4, 700)
    w = k.astype(np.float32)
    m, W = _model(spec, opts)
    with m:
        if kernel:
            assert m.kernel_name == kernel
        r = m.evaluate_result(f, sample_weight=w)
        d = m.evaluate_result(_dup(f, k))
        assert (r.rows, r.positives) == (700, int(np.asarray(f["label"]).sum()))
        assert (r.accuracy, r.roc_auc, r.pr_auc) == (d.accuracy, d.roc_auc, d.pr_auc)
        assert abs(r.loss * 700 / w.sum() - d.loss) <= 1e-6 * max(1.0, d.loss)
        _same(m.evaluate_result(f, sample_weight=np.ones(700, np.float32)), m.evaluate_result(f))
        rb = m.evaluate_result(f, batch_size=128, sample_weight=w)
        assert (rb.accuracy, rb.roc_auc, rb.pr_auc) == (r.accuracy, r.roc_auc, r.pr_auc)
        _same(m.evaluate_result(f, batch_size=128, sample_weight=w), rb)


@pytest.mark.gpu
def test_weighted_metrics_state():
    """srs_metrics_update_weighted_device: the trainer's weighted sums for the same rows, no mixing with unweighted
    updates until a reset, and the same bits on every run."""
    import torch
    from sparrowrecsys_b200.model import Metrics
    rng = np.random.default_rng(2)
    p = rng.random(5000).astype(np.float32)
    z = np.log(p / (1 - p)).astype(np.float32)
    y = (rng.random(5000) < 0.3).astype(np.int32)
    w = row_weights(5000, 2)
    dev = lambda a: torch.from_numpy(a).cuda()                              # noqa: E731
    ref = WO.keras_evaluate(p, z, y, w)
    results = []
    for _ in range(2):
        mt = Metrics(0)
        mt.update_device(dev(p[:3000]), dev(z[:3000]), dev(y[:3000]), weights=dev(w[:3000]))
        mt.update_device(dev(p[3000:]), dev(z[3000:]), dev(y[3000:]), weights=dev(w[3000:]))
        with pytest.raises(ValueError):
            mt.update_device(dev(p), dev(z), dev(y))
        results.append(mt.result())
        mt.reset()
        mt.update_device(dev(p), dev(z), dev(y))
        assert mt.result()["rows"] == 5000
        mt.close()
    for k in results[0]:
        assert np.array_equal(results[0][k], results[1][k]), k
    r = results[0]
    assert (r["accuracy"], r["roc_auc"], r["pr_auc"]) == pytest.approx(
        (ref["accuracy"], ref["roc_auc"], ref["pr_auc"]), rel=1e-12, abs=1e-15)
    assert r["loss"] == pytest.approx(ref["loss"], rel=1e-6)    # float32 log1p / exp per row differ by an ulp


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_rejections_leave_the_trainer_unchanged(model):
    from sparrowrecsys_b200 import _lib
    c = IDENTITY[model]
    W0, f, _ = _c_inputs(c)
    n = c.n
    bad = []
    for v in (-1.0, np.nan, np.inf):
        w = np.ones(n, np.float32)
        w[n // 2] = v
        bad.append(dict(sample_weight=w))
    bad += [dict(sample_weight=np.ones(n - 1, np.float32)), dict(class_weight={2: 1.0}),
            dict(class_weight={0: -1.0}),
            dict(validation_data=(f, f["label"], np.full(n, -1.0, np.float32)))]
    with _trainer(c, W0) as tr:
        tr.fit(f, epochs=1, batch_size=c.B, sample_weight=row_weights(n, 1))
        it, W1 = tr.iterations, tr.weights()
        for kw in bad:
            with pytest.raises(ValueError):
                tr.fit(f, epochs=1, batch_size=c.B, **kw)
            assert tr.iterations == it
            _same_weights(tr.weights(), W1)
        with pytest.raises(ValueError):
            tr.evaluate(f, sample_weight=np.full(n, np.nan, np.float32))
        # the library's own check, past the host helper
        keep = []
        batch, lab, _ = tr._rows(f, None, keep, "fit")
        order = np.arange(n, dtype=np.int32)
        w = np.ones(n, np.float32)
        w[-1] = -0.5
        hist = (_lib.SrsEvalResult * 1)()
        rc = tr._lib.srs_trainer_fit_weighted_host(tr._h, C.byref(batch), lab.ctypes.data, w.ctypes.data,
                                                   order.ctypes.data, c.B, 1, hist, None, None, None, 1, None)
        assert rc == _lib.SRS_ERR_INVALID
        assert tr.iterations == it
        _same_weights(tr.weights(), W1)


@pytest.mark.gpu
def test_dien_takes_no_weights():
    from sparrowrecsys_b200.training import Trainer
    from sparrowrecsys_b200.weights import init_aux_weights, init_weights
    spec = default_spec("dien", n_movies=50, n_users=60, emb_dim=8, hist_len=3)
    with Trainer(spec, {**init_weights(spec, 0), **init_aux_weights(spec, 0)}) as tr:
        with pytest.raises(NotImplementedError):
            tr.fit({}, sample_weight=[1.0])
        with pytest.raises(NotImplementedError):
            tr.fit({}, class_weight={0: 1.0})
        assert tr.iterations == 0
