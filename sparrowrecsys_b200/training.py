"""`model.fit` of NeuralCF, DeepFM, Wide&Deep, DeepFM_v2 and DIEN on the GPU (NeuralCF.py:74-91, DeepFM.py,
WideNDeep.py:99-117, DeepFM_v2.py:158-165: compile(loss='binary_crossentropy', optimizer='adam'), then
fit(train_dataset, epochs=5) over make_csv_dataset batches of 12), and of NeuralCF.py's second model, the two towers
(neural_cf_model_2 with its final Dense), compiled and fitted as its first.

    from sparrowrecsys_b200.training import Trainer
    tr = Trainer(spec, weights, device=0)                 # initial weights in Keras shapes
    history = tr.fit(train_features, epochs=5, batch_size=12, seed=0,
                     validation_data=test_features)       # optional: adds val_loss, val_accuracy, val_auc, val_auc_1
    loss, accuracy, roc_auc, pr_auc = tr.evaluate(test_features)   # the current weights, no export
    tr.fit(train_features, sample_weight=w, class_weight={0: 1.0, 1: 3.0})   # Keras's per-row weights
    model = tr.to_model()                                 # a serving CTRModel built from the trained weights

DIEN (DIEN.py:296-304: compile(optimizer="adam"), fit over batches of 12 with no shuffle) trains in file order
every epoch by default and reports its own history {"loss", "auc", "auc_value"} (section 4.20).

The forward, backward and Keras Adam run in the CUDA library (`srs_trainer_*`, include/srs_ctr.h; DESIGN.md
sections 4.8, 4.9, 4.18, 4.19, 4.20 and 4.27; sample weights 4.28).  For the other models TF's shuffle (buffer 10 000, unseeded) cannot be reproduced, so `fit` takes a seed instead: the host
draws one `numpy.random.default_rng(seed).permutation(n)` per epoch and the library trains in that row order.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Optional

import numpy as np

from . import _lib
from .features import _as_ids, encode_batch, negative_history_keys
from .model import CTRModel, _host_struct, _label_array, _spec_struct
from .spec import ModelSpec
from .weights import aux_weight_shapes, check_weights, weight_shapes


def sample_weights(labels, sample_weight=None, class_weight=None) -> Optional[np.ndarray]:
    """Keras's per-row weights (DESIGN.md section 4.28): w_i = sample_weight[i] * class_weight[label_i] in float32
    (a factor that is not given is 1), or None when neither is given.  `sample_weight` is [n] (or [n, 1]) numeric;
    `class_weight` maps the classes 0 and 1 to weights.  ValueError for a length other than the labels', a
    class_weight key other than 0 or 1, or a weight (given or multiplied) that is negative, NaN or infinite."""
    if sample_weight is None and class_weight is None:
        return None
    lab = np.asarray(labels).reshape(-1)
    n = lab.shape[0]
    w = np.ones(n, np.float32)
    if sample_weight is not None:
        sw = np.asarray(sample_weight)
        if sw.ndim == 2 and sw.shape[1] == 1:
            sw = sw[:, 0]
        if sw.ndim != 1 or sw.shape[0] != n:
            raise ValueError("sample_weight must be [%d] like the labels, got shape %s" % (n, sw.shape))
        if sw.dtype.kind not in "biuf":
            raise ValueError("sample_weight must be numeric")
        with np.errstate(over="ignore"):
            w = np.ascontiguousarray(sw, np.float32)
    if class_weight is not None:
        if not isinstance(class_weight, Mapping):
            raise ValueError("class_weight must map the classes 0 and 1 to weights")
        cw = np.ones(2, np.float32)
        for k, v in class_weight.items():
            if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or k not in (0, 1):
                raise ValueError("class_weight keys must be the classes 0 and 1, got %r" % (k,))
            with np.errstate(over="ignore"):
                cw[int(k)] = np.float32(v)
            if not (np.isfinite(cw[int(k)]) and cw[int(k)] >= 0):
                raise ValueError("class_weight[%d] is %r: weights must be finite and >= 0" % (int(k), v))
        with np.errstate(over="ignore", invalid="ignore"):
            w = w * np.where(lab == 1, cw[1], cw[0]).astype(np.float32)
    bad = ~(np.isfinite(w) & (w >= 0))
    if bad.any():
        i = int(np.argmax(bad))
        raise ValueError("the weight of row %d is %r: weights must be finite and >= 0" % (i, float(w[i])))
    return np.ascontiguousarray(w, np.float32)


def epoch_orders(n: int, epochs: int, seed: int) -> np.ndarray:
    """The row order of `Trainer.fit`: [epochs][n] int32, one `default_rng(seed).permutation(n)` per epoch."""
    rng = np.random.default_rng(seed)
    return np.stack([rng.permutation(n) for _ in range(int(epochs))]).astype(np.int32)


class Trainer:
    """Trainable NeuralCF, two-tower, DeepFM, Wide&Deep, DeepFM_v2 or DIEN weights and Keras Adam's state on one
    GPU."""

    MODELS = ("neuralcf", "twotowers", "deepfm", "widendeep", "deepfm_v2", "dien")

    def __init__(self, spec: ModelSpec, weights: Mapping[str, np.ndarray], device: int = 0,
                 adam: Optional[Mapping[str, float]] = None):
        """`weights`: the initial weights (canonical names, Keras shapes, float32 host arrays), e.g.
        `init_weights(spec, seed, for_test=False)` for an untrained model.  `adam`: Keras Adam's lr, beta_1,
        beta_2, epsilon (default: Keras's 0.001, 0.9, 0.999, 1e-7).  DIEN's weights include the auxiliary head's
        group (`weights.init_aux_weights`): its objective needs them.  The two towers train only with their final
        Dense (`spec.final_dense`; without it the output is the raw Dot, which binary cross-entropy does not take:
        ValueError).  NotImplementedError for any model but NeuralCF, two towers, DeepFM, Wide&Deep, DeepFM_v2
        and DIEN."""
        if spec.model not in self.MODELS:
            raise NotImplementedError("fit is implemented for NeuralCF (neural_cf_model_1), two towers "
                                      "(neural_cf_model_2), DeepFM, Wide&Deep, DeepFM_v2 and DIEN only, not %r"
                                      % spec.model)
        self.spec = spec
        self.device = int(device)
        self._h = None
        self._lib = _lib.load()
        check_weights(spec, weights)
        shapes = _shapes(spec)
        tensors = (_lib.SrsTensor * len(shapes))()
        keep = []
        for i, (name, shape) in enumerate(shapes):
            a = np.ascontiguousarray(weights[name], np.float32)
            keep.append(a)
            tensors[i] = _lib.SrsTensor(name.encode(), a.ctypes.data, shape[0], shape[1] if len(shape) > 1 else 1,
                                        _lib.SRS_HOST)
        hp = None
        if adam is not None:
            d = {"lr": 0.001, "beta_1": 0.9, "beta_2": 0.999, "epsilon": 1e-7}
            d.update(adam)
            hp = C.byref(_lib.SrsAdam(d["lr"], d["beta_1"], d["beta_2"], d["epsilon"]))
        h = C.c_void_p()
        sp = _spec_struct(spec)
        _lib.check(self._lib.srs_trainer_create_any(C.byref(sp), tensors, len(shapes), self.device, hp, C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.srs_trainer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def iterations(self) -> int:
        """Adam steps taken so far (Keras's `optimizer.iterations`)."""
        return int(self._lib.srs_trainer_iterations(self._h))

    def fit(self, features: Mapping[str, object], labels=None, epochs: int = 5, batch_size: int = 12, seed: int = 0,
            order=None, validation_data=None, validation_split: float = 0.0,
            validation_freq: int = 1, sample_weight=None, class_weight=None) -> Dict[str, list]:
        """`model.fit(dataset, epochs)`: train on the rows of `features` (the model's `predict` columns: `movieId`,
        `userId` for NeuralCF and two towers, also the 7 numerics, `movieGenre1` and `userGenre1` for DeepFM and DeepFM_v2, the 7 numerics, all eight
        genre columns and `userRatedMovie1` for Wide&Deep; labels default to
        `features["label"]`) in batches of `batch_size`, the last one partial.  The row order of epoch e is
        `epoch_orders(n, epochs, seed)[e]` unless `order` ([epochs][n], each a permutation) is given.  Returns
        Keras's history dict {"loss", "accuracy", "auc", "auc_1"}: one value per epoch, each computed on the
        steps' forward outputs before their updates (`auc` ROC, `auc_1` PR, the compile line's metric names).
        ValueError for an out-of-range id or genre, a label other than 0 / 1, or a bad order, KeyError for a
        missing column; the weights are then unchanged.

        DIEN: `features` also carries `negtive_userRatedMovie2..T` (a missing one is a KeyError, as in
        `CTRModel.dien_outputs`); the row order defaults to file order every epoch (DIEN.py's dataset has no
        shuffle; `seed` is not used), an explicit `order` is still taken; the history is {"loss", "auc",
        "auc_value"}, each epoch's as `CTRModel.dien_evaluate` defines them over the steps' outputs; validation is
        not supported (NotImplementedError).

        Validation, as Keras's `fit`: `validation_data` is `(x_val, y_val)` or a feature dict with "label";
        otherwise `validation_split` = f in (0, 1) holds out the last floor(n * f) rows, taken before any
        shuffling (training then uses the first n - floor(n * f) rows, and `order` is over those).  The epochs e
        with (e + 1) % `validation_freq` == 0 end, after their last update, with `evaluate` of the current weights
        on the validation rows (one batch, in file order), logged as "val_loss", "val_accuracy", "val_auc" and
        "val_auc_1" for those epochs only.  Validation changes no weight, no Adam state and no training log.  Its
        rows are checked like the training rows before anything runs.

        Weights, as Keras's (DESIGN.md section 4.28): `sample_weight` [n] and `class_weight` {0: w0, 1: w1} weight
        row i by sample_weight[i] * class_weight[label_i] (`sample_weights`).  A step's loss is then
        sum w_i l_i / B, and the history's metrics are weighted.  `class_weight` applies to the training rows only;
        `validation_data` may be `(x_val, y_val, val_sample_weight)`, and `validation_split` splits `sample_weight`
        with the rows.  Weights are checked before anything runs.  DIEN: NotImplementedError (its loss carries the
        auxiliary term)."""
        if self.spec.model == "dien":
            if sample_weight is not None or class_weight is not None:
                raise NotImplementedError("DIEN's fit takes no sample_weight or class_weight: its loss carries the "
                                          "auxiliary negative-sample term")
            if validation_data is not None or validation_split or validation_freq != 1:
                raise NotImplementedError("DIEN's fit takes no validation: DIEN.py validates nothing during fit")
            return self._fit_dien(features, labels, epochs, batch_size, order)
        res, vres, validated = self._fit(features, labels, epochs, batch_size, seed, order, validation_data,
                                         validation_split, validation_freq, sample_weight, class_weight)
        out = _logs(res, "")
        if validated:
            out.update(_logs([vres[e] for e in validated], "val_"))
        return out

    def _fit(self, features, labels=None, epochs=5, batch_size=12, seed=0, order=None, validation_data=None,
             validation_split=0.0, validation_freq=1, sample_weight=None, class_weight=None):
        """`fit`, returning the library's results: (the epochs' srs_eval_result, the validation's [epochs] with
        zeroed entries for epochs not validated, the validated epochs)."""
        val, val_sw = None, None
        if validation_data is not None:
            val, val_sw = _validation_triple(validation_data)
        elif validation_split:
            split = float(validation_split)
            if not 0.0 < split < 1.0:
                raise ValueError("validation_split must be in (0, 1), got %r" % (validation_split,))
            lab = _label_array(features, labels)
            n = lab.shape[0]
            split_at = int(np.floor(n * (1.0 - split)))       # Keras's train_validation_split
            if split_at == 0 or split_at == n:
                raise ValueError("%d rows are not enough to split into a training and a validation part with "
                                 "validation_split=%r" % (n, validation_split))
            val = (_take(features, split_at, n), lab[split_at:])
            features, labels = _take(features, 0, split_at), lab[:split_at]
            if sample_weight is not None:                     # split with the rows, checked over all n first
                sw = sample_weights(lab, sample_weight)
                sample_weight, val_sw = sw[:split_at], sw[split_at:]
        if isinstance(validation_freq, bool) or not isinstance(validation_freq, (int, np.integer)) \
                or validation_freq < 1:
            raise ValueError("validation_freq must be an integer >= 1, got %r" % (validation_freq,))
        keep = []
        batch, lab, n = self._rows(features, labels, keep, "fit")
        w = sample_weights(lab, sample_weight, class_weight)
        epochs, batch_size = int(epochs), int(batch_size)
        if order is None:
            order = epoch_orders(n, epochs, seed)
        order = np.ascontiguousarray(order, np.int32)
        if order.shape != (epochs, n):
            raise ValueError("order must be [epochs=%d][n=%d], got %s" % (epochs, n, order.shape))
        hist = (_lib.SrsEvalResult * max(epochs, 1))()
        vhist = (_lib.SrsEvalResult * max(epochs, 1))()
        vbatch, vlab, vw = None, None, None
        if val is not None:
            vb, vlab, _ = self._rows(val[0], val[1], keep, "validation")
            vbatch = C.byref(vb)
            vw = sample_weights(vlab, val_sw)                 # class_weight is for the training rows only
        if w is None and vw is None:
            _lib.check(self._lib.srs_trainer_fit_validate_host(
                self._h, C.byref(batch), lab.ctypes.data, order.ctypes.data, batch_size, epochs, hist, vbatch,
                None if vlab is None else vlab.ctypes.data, int(validation_freq), vhist))
        else:
            _lib.check(self._lib.srs_trainer_fit_weighted_host(
                self._h, C.byref(batch), lab.ctypes.data, None if w is None else w.ctypes.data, order.ctypes.data,
                batch_size, epochs, hist, vbatch, None if vlab is None else vlab.ctypes.data,
                None if vw is None else vw.ctypes.data, int(validation_freq), vhist))
        validated = [e for e in range(epochs) if val is not None and (e + 1) % validation_freq == 0]
        return list(hist[:epochs]), list(vhist[:epochs]), validated

    def _fit_dien(self, features, labels, epochs, batch_size, order) -> Dict[str, list]:
        """DIEN's fit: the rows, their negatives and labels to srs_trainer_fit_dien_host."""
        keep = []
        batch, lab, n = self._rows(features, labels, keep, "fit")
        keys = negative_history_keys(self.spec.hist_len)
        neg = np.empty((n, max(len(keys), 1)), np.int32)
        for j, k in enumerate(keys):
            neg[:, j] = _as_ids(features, k, self.spec.n_movies, "negative movie id")
        neg = np.ascontiguousarray(neg[:, :len(keys)])
        epochs, batch_size = int(epochs), int(batch_size)
        if order is None:
            order = np.tile(np.arange(n, dtype=np.int32), (epochs, 1))
        order = np.ascontiguousarray(order, np.int32)
        if order.shape != (epochs, n):
            raise ValueError("order must be [epochs=%d][n=%d], got %s" % (epochs, n, order.shape))
        hist = (_lib.SrsDienEvalResult * max(epochs, 1))()
        _lib.check(self._lib.srs_trainer_fit_dien_host(
            self._h, C.byref(batch), neg.ctypes.data if neg.size else None, neg.shape[1], lab.ctypes.data,
            order.ctypes.data, batch_size, epochs, hist))
        res = list(hist[:epochs])
        return {"loss": [r.loss for r in res], "auc": [r.auc for r in res], "auc_value": [r.auc_value for r in res]}

    def evaluate(self, features: Mapping[str, object], labels=None, sample_weight=None):
        """`model.evaluate(x)` of the current weights: (loss, accuracy, roc_auc, pr_auc) over the rows of
        `features` in one batch, as `CTRModel.evaluate` of `to_model()` reports them (on CUDA cores), without
        exporting the weights; weighted by `sample_weight` [n] when given (DESIGN.md section 4.28).  Errors as
        `fit`'s.  DIEN: NotImplementedError, as `tfrecmodel.dien.evaluate`: its Keras evaluate is
        `to_model().dien_evaluate`."""
        if self.spec.model == "dien":
            raise NotImplementedError("DIEN's Keras evaluate reports the loss with the auxiliary negative-sample term "
                                      "and its AUC metrics, not the four compile metrics; use "
                                      "Trainer.to_model().dien_evaluate")
        r = self.evaluate_result(features, labels, sample_weight)
        return r.loss, r.accuracy, r.roc_auc, r.pr_auc

    def evaluate_result(self, features, labels=None, sample_weight=None) -> _lib.SrsEvalResult:
        """`evaluate` with the counts: the `srs_eval_result` (rows, positives, correct and the four metrics)."""
        keep = []
        batch, lab, _ = self._rows(features, labels, keep, "evaluate")
        w = sample_weights(lab, sample_weight)
        out = _lib.SrsEvalResult()
        if w is None:
            _lib.check(self._lib.srs_trainer_evaluate_host(self._h, C.byref(batch), lab.ctypes.data, C.byref(out)))
        else:
            _lib.check(self._lib.srs_trainer_evaluate_weighted_host(self._h, C.byref(batch), lab.ctypes.data,
                                                                    w.ctypes.data, C.byref(out)))
        return out

    def _rows(self, features, labels, keep: list, what: str):
        """(srs_batch over host arrays kept alive in `keep`, int32 labels, rows) of the model's columns."""
        lab = _label_array(features, labels)
        n = lab.shape[0]
        if self.spec.model in ("neuralcf", "twotowers"):
            movie = _ids(features, "movieId")
            user = _ids(features, "userId")
            if movie.shape[0] != n or user.shape[0] != n:
                raise ValueError("labels have %d rows, the features %d" % (n, movie.shape[0]))
            keep += [movie, user]
            batch = _lib.SrsBatch(n, 0, movie.ctypes.data, user.ctypes.data, None, None, None, None, None)
        else:                                           # predict's encoding: keys, dtypes, genre strings, errors
            enc = encode_batch(self.spec, features)
            if enc.B != n:
                raise ValueError("labels have %d rows, the features %d" % (n, enc.B))
            batch = _host_struct(enc, keep)
        if n == 0:
            raise ValueError("%s needs at least one row" % what)
        keep.append(lab)
        return batch, lab, n

    def weights(self) -> Dict[str, np.ndarray]:
        """The current weights, canonical names and Keras shapes (float32 host arrays)."""
        out = {}
        for name, shape in _shapes(self.spec):
            a = np.empty(shape, np.float32)
            _lib.check(self._lib.srs_trainer_get_weights(self._h, name.encode(), a.ctypes.data))
            out[name] = a
        return out

    def to_model(self, device: Optional[int] = None) -> CTRModel:
        """A serving `CTRModel` built from the current weights (the trainer is not shared with it)."""
        return CTRModel(self.spec, self.weights(), self.device if device is None else device)


def _shapes(spec: ModelSpec):
    """The trainer's tensors: the model's, and for DIEN the auxiliary head's group, which its objective needs."""
    return weight_shapes(spec) + (aux_weight_shapes(spec) if spec.model == "dien" else [])


def _logs(results, prefix: str) -> Dict[str, list]:
    """Keras's History lists of srs_eval_results: loss, accuracy, auc (ROC), auc_1 (PR)."""
    return {prefix + "loss": [r.loss for r in results], prefix + "accuracy": [r.accuracy for r in results],
            prefix + "auc": [r.roc_auc for r in results], prefix + "auc_1": [r.pr_auc for r in results]}


def _validation_pair(validation_data):
    """(features, labels) of `validation_data`: `(x_val, y_val)`, or a feature dict whose "label" holds the labels."""
    if isinstance(validation_data, Mapping):
        return validation_data, None
    if isinstance(validation_data, (tuple, list)) and len(validation_data) == 2 \
            and isinstance(validation_data[0], Mapping):
        return validation_data[0], validation_data[1]
    raise ValueError("validation_data must be (features, labels) or a feature dict with 'label'")


def _validation_triple(validation_data):
    """(features, labels, sample_weight or None) of `validation_data`: `_validation_pair`'s forms, or
    `(x_val, y_val, val_sample_weight)`."""
    if isinstance(validation_data, (tuple, list)) and len(validation_data) == 3 \
            and isinstance(validation_data[0], Mapping):
        return (validation_data[0], validation_data[1]), validation_data[2]
    return _validation_pair(validation_data), None


def _take(features, lo: int, hi: int) -> Dict[str, np.ndarray]:
    """Rows lo .. hi of every column of a feature dict."""
    return {k: np.asarray(v)[lo:hi] for k, v in features.items()}


def _ids(features, key) -> np.ndarray:
    if key not in features:
        raise KeyError("missing required feature %r" % key)
    a = np.asarray(features[key])
    if a.ndim == 2 and a.shape[1] == 1:
        a = a[:, 0]
    if a.ndim != 1 or a.dtype.kind not in "iu":
        raise ValueError("%s must be a 1-D integer column" % key)
    if a.size and (a.min() < np.iinfo(np.int32).min or a.max() > np.iinfo(np.int32).max):
        raise ValueError("%s is outside the int32 range" % key)
    return np.ascontiguousarray(a, np.int32)            # the library range-checks against the vocabulary
