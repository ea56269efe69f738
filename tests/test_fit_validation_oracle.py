"""CPU checks of validation during `fit` (DESIGN.md section 4.10): the oracle's epoch-by-epoch validated fit
(oracle/fit_validation.py) against the one-call fits of oracle/ncf_train.py and oracle/deepfm_train.py, and the
rejections that `Trainer.fit` and the ABI make before any device call."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import deepfm_train, fit_validation, keras_eval, ncf_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _data(model, n, nv):
    """n training rows and the next nv rows as validation, from the model's training set."""
    z = dict(np.load(os.path.join(GOLDEN, "%s_trainset.npz" % model)))
    train = {k: np.ascontiguousarray(v[:n]) for k, v in z.items()}
    val = {k: np.ascontiguousarray(v[n:n + nv]) for k, v in z.items()}
    return train, val


def _one_call(model, W0, f, orders, B, dtype):
    if model == "neuralcf":
        return ncf_train.fit(W0, f["movieId"], f["userId"], f["label"], orders, B, dtype)
    return deepfm_train.fit(W0, deepfm_train.Rows.from_features(f), f["label"], orders, B, dtype)


def _same_bits(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("model", ["neuralcf", "deepfm"])
def test_epoch_by_epoch_is_one_multi_epoch_fit(model, dtype):
    """Weights, Adam's m, v and iterations, and the history: the same numpy bits."""
    W0 = init_weights(default_spec(model), 2, for_test=False)
    f, _ = _data(model, 90, 0)
    orders = ncf_train.epoch_orders(90, 3, 4)
    W1, h1, _, opt1 = _one_call(model, W0, f, orders, 12, dtype)
    W, opt, hist = W0, None, []
    for e in range(3):
        W, h, vh, opt = fit_validation.fit(model, W, f, orders[e:e + 1], 12, dtype, opt=opt)
        assert vh == [None]
        hist += h
    _same_bits(W, W1)
    _same_bits(opt.m, opt1.m)
    _same_bits(opt.v, opt1.v)
    assert opt.iterations == opt1.iterations == 3 * 8
    assert hist == h1


@pytest.mark.parametrize("model", ["neuralcf", "deepfm"])
def test_validation_reads_the_weights_only_and_evaluates_them(model):
    """With validation the weights, Adam state and training history keep their bits; each validated epoch's entry is
    keras_evaluate of the forward of the validation rows under that epoch's weights."""
    W0 = init_weights(default_spec(model), 3, for_test=False)
    f, val = _data(model, 60, 40)
    orders = ncf_train.epoch_orders(60, 4, 1)
    W, h, vh, opt = fit_validation.fit(model, W0, f, orders, 33, np.float32, val=val, validation_freq=2)
    Wn, hn, vhn, optn = fit_validation.fit(model, W0, f, orders, 33, np.float32)
    _same_bits(W, Wn)
    _same_bits(opt.m, optn.m)
    assert h == hn and vhn == [None] * 4
    assert vh[0] is None and vh[2] is None
    Wp = init_weights(default_spec(model), 3, for_test=False)
    opt_e = None
    for e in range(4):
        Wp, _, _, opt_e = fit_validation.fit(model, Wp, f, orders[e:e + 1], 33, np.float32, opt=opt_e)
        if (e + 1) % 2:
            continue
        if model == "neuralcf":
            p, z, _ = ncf_train.forward(Wp, val["movieId"], val["userId"], np.float32)
        else:
            p, z, _ = deepfm_train.forward(Wp, deepfm_train.Rows.from_features(val), np.float32)
        r = keras_eval.keras_evaluate(p, z, val["label"])
        assert vh[e] == {k: r[k] for k in fit_validation.METRICS}, e


# ---- rejections before any device call -------------------------------------------------------------------------
class _NoDevice:
    """A library stand-in that fails the test if anything reaches it."""

    def __getattr__(self, name):
        raise AssertionError("%s was called" % name)


def _trainer(model):
    from sparrowrecsys_b200.training import Trainer
    tr = Trainer.__new__(Trainer)
    tr.spec, tr.device, tr._h, tr._lib = default_spec(model), 0, None, _NoDevice()
    return tr


@pytest.mark.parametrize("split", [-0.25, 1.0, 1.5, float("nan")])
def test_bad_validation_split_is_a_value_error(split):
    f, _ = _data("neuralcf", 20, 0)
    with pytest.raises(ValueError, match="validation_split"):
        _trainer("neuralcf").fit(f, epochs=1, validation_split=split)


@pytest.mark.parametrize("n,split", [(3, 1e-17), (3, 0.99), (1, 0.5)])
def test_validation_split_with_an_empty_part_is_a_value_error(n, split):
    """Keras's split_at = floor(n (1 - f)): 0 or n leaves one part empty (1 - 1e-17 is 1.0 in double)."""
    f, _ = _data("neuralcf", n, 0)
    with pytest.raises(ValueError, match="not enough to split"):
        _trainer("neuralcf").fit(f, epochs=1, validation_split=split)


@pytest.mark.parametrize("freq", [0, -1, 1.5, True, [1, 2]])
def test_bad_validation_freq_is_a_value_error(freq):
    f, val = _data("neuralcf", 20, 10)
    with pytest.raises(ValueError, match="validation_freq"):
        _trainer("neuralcf").fit(f, epochs=1, validation_data=val, validation_freq=freq)


@pytest.mark.parametrize("bad", [(1, 2), ({"movieId": np.zeros(1, np.int32)},), [np.zeros(3)], "test.csv"])
def test_validation_data_must_be_a_pair_or_a_labelled_dict(bad):
    f, _ = _data("neuralcf", 20, 0)
    with pytest.raises(ValueError, match="validation_data"):
        _trainer("neuralcf").fit(f, epochs=1, validation_data=bad)


def test_validation_rows_missing_a_column_or_label_are_rejected_before_the_library():
    f, val = _data("deepfm", 20, 10)
    with pytest.raises(KeyError, match="userRatingStddev"):
        _trainer("deepfm").fit(f, epochs=1, validation_data={k: v for k, v in val.items() if k != "userRatingStddev"})
    with pytest.raises(KeyError, match="label"):
        _trainer("deepfm").fit(f, epochs=1, validation_data={k: v for k, v in val.items() if k != "label"})
    with pytest.raises(ValueError, match="rows"):
        _trainer("deepfm").fit(f, epochs=1, validation_data=(val, val["label"][:5]))


def test_abi_validation_entry_points_reject_null_arguments():
    from sparrowrecsys_b200 import _lib
    try:
        lib = _lib.load()
    except ImportError as e:
        pytest.skip(str(e))
    r = _lib.SrsEvalResult()
    b = _lib.SrsBatch()
    assert lib.srs_trainer_evaluate_host(None, C.byref(b), None, C.byref(r)) == _lib.SRS_ERR_INVALID
    assert lib.srs_trainer_fit_validate_host(None, C.byref(b), None, None, 12, 1, None, C.byref(b), None, 1,
                                             None) == _lib.SRS_ERR_INVALID
