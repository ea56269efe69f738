"""`model.fit` of NeuralCF and DeepFM on the GPU (NeuralCF.py:74-91, DeepFM.py: compile(loss='binary_crossentropy',
optimizer='adam'), then fit(train_dataset, epochs=5) over make_csv_dataset batches of 12).

    from sparrowrecsys_b200.training import Trainer
    tr = Trainer(spec, weights, device=0)                 # initial weights in Keras shapes
    history = tr.fit(train_features, epochs=5, batch_size=12, seed=0)
    model = tr.to_model()                                 # a serving CTRModel built from the trained weights

The forward, backward and Keras Adam run in the CUDA library (`srs_trainer_*`, include/srs_ctr.h; DESIGN.md
sections 4.8 and 4.9).  TF's shuffle (buffer 10 000, unseeded) cannot be reproduced, so `fit` takes a seed instead: the host
draws one `numpy.random.default_rng(seed).permutation(n)` per epoch and the library trains in that row order.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Optional

import numpy as np

from . import _lib
from .features import encode_batch
from .model import CTRModel, _host_struct, _label_array, _spec_struct
from .spec import ModelSpec
from .weights import check_weights, weight_shapes


def epoch_orders(n: int, epochs: int, seed: int) -> np.ndarray:
    """The row order of `Trainer.fit`: [epochs][n] int32, one `default_rng(seed).permutation(n)` per epoch."""
    rng = np.random.default_rng(seed)
    return np.stack([rng.permutation(n) for _ in range(int(epochs))]).astype(np.int32)


class Trainer:
    """Trainable NeuralCF or DeepFM weights and Keras Adam's state on one GPU."""

    MODELS = ("neuralcf", "deepfm")

    def __init__(self, spec: ModelSpec, weights: Mapping[str, np.ndarray], device: int = 0,
                 adam: Optional[Mapping[str, float]] = None):
        """`weights`: the initial weights (canonical names, Keras shapes, float32 host arrays), e.g.
        `init_weights(spec, seed, for_test=False)` for an untrained model.  `adam`: Keras Adam's lr, beta_1,
        beta_2, epsilon (default: Keras's 0.001, 0.9, 0.999, 1e-7).  NotImplementedError for any model but
        NeuralCF and DeepFM."""
        if spec.model not in self.MODELS:
            raise NotImplementedError("fit is implemented for NeuralCF (neural_cf_model_1) and DeepFM only, not %r"
                                      % spec.model)
        self.spec = spec
        self.device = int(device)
        self._h = None
        self._lib = _lib.load()
        check_weights(spec, weights)
        shapes = weight_shapes(spec)
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
        _lib.check(self._lib.srs_trainer_create(C.byref(sp), tensors, len(shapes), self.device, hp, C.byref(h)))
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
            order=None) -> Dict[str, list]:
        """`model.fit(dataset, epochs)`: train on the rows of `features` (the model's `predict` columns: `movieId`,
        `userId` for NeuralCF, also the 7 numerics, `movieGenre1` and `userGenre1` for DeepFM; labels default to
        `features["label"]`) in batches of `batch_size`, the last one partial.  The row order of epoch e is
        `epoch_orders(n, epochs, seed)[e]` unless `order` ([epochs][n], each a permutation) is given.  Returns
        Keras's history dict {"loss", "accuracy", "auc", "auc_1"}: one value per epoch, each computed on the
        steps' forward outputs before their updates (`auc` ROC, `auc_1` PR, the compile line's metric names).
        ValueError for an out-of-range id or genre, a label other than 0 / 1, or a bad order, KeyError for a
        missing column; the weights are then unchanged."""
        lab = _label_array(features, labels)
        n = lab.shape[0]
        keep = []
        if self.spec.model == "neuralcf":
            movie = _ids(features, "movieId")
            user = _ids(features, "userId")
            if movie.shape[0] != n or user.shape[0] != n:
                raise ValueError("labels have %d rows, the features %d" % (n, movie.shape[0]))
            batch = _lib.SrsBatch(n, 0, movie.ctypes.data, user.ctypes.data, None, None, None, None, None)
        else:                                           # predict's encoding: keys, dtypes, genre strings, errors
            enc = encode_batch(self.spec, features)
            if enc.B != n:
                raise ValueError("labels have %d rows, the features %d" % (n, enc.B))
            batch = _host_struct(enc, keep)
        if n == 0:
            raise ValueError("fit needs at least one row")
        epochs, batch_size = int(epochs), int(batch_size)
        if order is None:
            order = epoch_orders(n, epochs, seed)
        order = np.ascontiguousarray(order, np.int32)
        if order.shape != (epochs, n):
            raise ValueError("order must be [epochs=%d][n=%d], got %s" % (epochs, n, order.shape))
        hist = (_lib.SrsEvalResult * max(epochs, 1))()
        _lib.check(self._lib.srs_trainer_fit_host(self._h, C.byref(batch), lab.ctypes.data, order.ctypes.data,
                                                  batch_size, epochs, hist))
        return {"loss": [h.loss for h in hist[:epochs]], "accuracy": [h.accuracy for h in hist[:epochs]],
                "auc": [h.roc_auc for h in hist[:epochs]], "auc_1": [h.pr_auc for h in hist[:epochs]]}

    def weights(self) -> Dict[str, np.ndarray]:
        """The current weights, canonical names and Keras shapes (float32 host arrays)."""
        out = {}
        for name, shape in weight_shapes(self.spec):
            a = np.empty(shape, np.float32)
            _lib.check(self._lib.srs_trainer_get_weights(self._h, name.encode(), a.ctypes.data))
            out[name] = a
        return out

    def to_model(self, device: Optional[int] = None) -> CTRModel:
        """A serving `CTRModel` built from the current weights (the trainer is not shared with it)."""
        return CTRModel(self.spec, self.weights(), self.device if device is None else device)


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
