"""CPU oracle of Keras's `fit(..., validation_data=..., validation_freq=...)` for NeuralCF and DeepFM.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

The epochs run one at a time from `oracle.ncf_train` / `oracle.deepfm_train`'s step functions (`gradients`, `Adam`)
and the Adam state carries over from one call to the next, so a fit can be continued.  After every epoch e with
(e + 1) % validation_freq == 0 the validation rows go through the model's `forward` at the fit's dtype and
`keras_eval.keras_evaluate` (DESIGN.md section 4.10).  Validation reads the weights only.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np

from . import deepfm_train, keras_eval, ncf_train

METRICS = ("loss", "accuracy", "roc_auc", "pr_auc")


def _summary(p, z, y) -> dict:
    r = keras_eval.keras_evaluate(np.asarray(p).astype(np.float32), np.asarray(z).astype(np.float32), np.asarray(y))
    return {k: r[k] for k in METRICS}


class _NeuralCF:
    Adam = ncf_train.Adam

    def __init__(self, features):
        self.movie = np.asarray(features["movieId"])
        self.user = np.asarray(features["userId"])

    def step(self, W, opt, rows, y, dtype):
        mid, uid = self.movie[rows], self.user[rows]
        g, p, z = ncf_train.gradients(W, mid, uid, y, dtype)
        opt.step(W, g, {"movieId_embedding": mid, "userId_embedding": uid})
        return p, z

    def forward(self, W, dtype):
        p, z, _ = ncf_train.forward(W, self.movie, self.user, dtype)
        return p, z


class _DeepFM:
    Adam = deepfm_train.Adam

    def __init__(self, features):
        self.rows = deepfm_train.Rows.from_features(features)

    def step(self, W, opt, rows, y, dtype):
        r = self.rows.take(rows)
        g, p, z = deepfm_train.gradients(W, r, y, dtype)
        opt.step(W, g, deepfm_train.table_rows(r))
        return p, z

    def forward(self, W, dtype):
        p, z, _ = deepfm_train.forward(W, self.rows, dtype)
        return p, z


MODELS = {"neuralcf": _NeuralCF, "deepfm": _DeepFM}


def fit(model: str, W, features, orders, batch_size: int, dtype=np.float32, val=None, validation_freq: int = 1,
        opt=None, hp=None):
    """`model.fit` of `model` ("neuralcf" or "deepfm") over the rows of the feature dict `features` (labels in
    "label") in the row orders `orders` [epochs][n], batches of `batch_size`, the last one partial, with Keras Adam
    (`hp`); `val`: None or a feature dict of validation rows.  `opt`: the Adam state of an earlier call to continue
    from (None: a fresh one, with iterations 0).  Returns (weights at `dtype`, history, val_history, Adam):

    * history: per epoch, keras_evaluate of the steps' outputs before their updates (as `ncf_train.fit`);
    * val_history: per epoch, keras_evaluate of the forward of `val` after the epoch's last update for a validated
      epoch, None for the others.
    Epoch by epoch, continuing with `opt`, gives the bits of one call over all the epochs."""
    m = MODELS[model](features)
    label = np.asarray(features["label"])
    W = ncf_train.as_dtype(W, dtype)
    if opt is None:
        opt = m.Adam(W, dtype, hp)
    v = None if val is None else MODELS[model](val)
    history: List[dict] = []
    val_history: List[Optional[dict]] = []
    for e, order in enumerate(orders):
        ps, zs, ys = [], [], []
        for lo in range(0, len(order), batch_size):
            rows = np.asarray(order[lo:lo + batch_size])
            y = label[rows]
            p, z = m.step(W, opt, rows, y, dtype)
            ps.append(p); zs.append(z); ys.append(y)
        history.append(_summary(np.concatenate(ps), np.concatenate(zs), np.concatenate(ys)))
        if v is not None and (e + 1) % validation_freq == 0:
            p, z = v.forward(W, dtype)
            val_history.append(_summary(p, z, val["label"]))
        else:
            val_history.append(None)
    return W, history, val_history, opt
