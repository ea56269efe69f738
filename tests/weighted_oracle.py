"""CPU oracle of Keras's `sample_weight` / `class_weight` in `fit` and `evaluate` (DESIGN.md section 4.28), on top of
the unweighted oracles, which it leaves as they are.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

* `keras_evaluate(probs, logits, labels, sample_weight)`: `oracle.keras_eval.keras_evaluate` with weighted metrics.
  Row i counts as w_i in TP/FP/TN/FN (float64 sums), accuracy is sum w_i [correct_i] / sum w_i (0 when the weights
  sum to 0) and loss sum w_i l_i / rows, with w_i l_i in float32 (SUM_OVER_BATCH_SIZE).  rows, positives and correct
  stay counts.
* `gradients(model, W, *columns, y, dtype, weight=w)`: the model oracle's `gradients` with dL/dz_i =
  (w_i (p_i - y_i)) / B, in that order, so that w = 1 gives the unweighted values bit for bit.  Every training oracle
  computes dz = (p - y) / B from the `p` of its module's `forward`; for the call, that `forward` is wrapped so that
  its `p`, subtracted from the labels, gives `numerator(p, y, w, dtype)` = w (p - y) instead.  Everything else is
  the model oracle's own backward.
* `fit(model, W, data, label, orders, batch_size, dtype, hp=None, weights=None)`: the model oracle's `fit` loop
  with the dataset's row weights `weights` [n]; returns (weights at `dtype`, history).
"""
from __future__ import annotations

import numpy as np

from oracle import deepfm_train, deepfm_v2_train, keras_eval, ncf_train, twotowers_train, widendeep_train

ORACLE = {"neuralcf": ncf_train, "twotowers": twotowers_train, "deepfm": deepfm_train, "widendeep": widendeep_train,
          "deepfm_v2": deepfm_v2_train}


def numerator(p, y, w, dtype):
    """A weighted step's dL/dz times B: w (p - y), each operation rounded at `dtype`."""
    g = (np.asarray(p) - np.asarray(y).astype(dtype)).astype(dtype)
    return (np.asarray(w).astype(dtype) * g).astype(dtype)


class _WeightedProbs(np.ndarray):
    """Probabilities whose difference with the labels is `numerator(p, y, w, dtype)`."""

    def __sub__(self, y):
        return numerator(self.view(np.ndarray), y, self.weight, self.step_dtype)


def gradients(model, W, *args, weight=None):
    """(grads, p, z) of `ORACLE[model].gradients(W, *args)` with row weights `weight` (None: unweighted).  `args`
    are the model oracle's: the columns (or Rows), the labels and the dtype."""
    mod = ORACLE[model]
    if weight is None:
        return mod.gradients(W, *args)
    dtype = args[-1] if len(args) > 0 and isinstance(args[-1], type) else np.float32
    intact = mod.forward

    def forward(*a, **kw):
        p, z, cache = intact(*a, **kw)
        wp = np.asarray(p).view(_WeightedProbs)
        wp.weight, wp.step_dtype = weight, dtype
        return wp, z, cache

    mod.forward = forward
    try:
        g, p, z = mod.gradients(W, *args)
    finally:
        mod.forward = intact
    return g, np.asarray(p).view(np.ndarray), z


def weighted_confusion(probs, labels, weights):
    """(tp, fp, tn, fn), float64 [200] each: `keras_eval.confusion_counts` with row i counted as weights[i]."""
    p = np.asarray(probs, np.float32).reshape(-1)
    pos = np.asarray(labels).reshape(-1) != 0
    w = np.asarray(weights, np.float32).astype(np.float64).reshape(-1)
    pred = p[:, None] > keras_eval.keras_thresholds()[None, :]
    tp = (pred & pos[:, None]).astype(np.float64).T @ w
    fp = (pred & ~pos[:, None]).astype(np.float64).T @ w
    fn = (~pred & pos[:, None]).astype(np.float64).T @ w
    tn = (~pred & ~pos[:, None]).astype(np.float64).T @ w
    return tp, fp, tn, fn


def keras_evaluate(probs, logits, labels, sample_weight=None) -> dict:
    """`keras_eval.keras_evaluate`, weighted by `sample_weight` [rows] (finite, >= 0) when given."""
    if sample_weight is None:
        return keras_eval.keras_evaluate(probs, logits, labels)
    r = keras_eval.keras_evaluate(probs, logits, labels)          # its checks, rows, positives and correct
    p = np.asarray(probs, np.float32).reshape(-1)
    lab = np.asarray(labels).reshape(-1)
    w = np.asarray(sample_weight, np.float32).reshape(-1)
    if w.shape[0] != p.shape[0] or not np.all(np.isfinite(w) & (w >= 0)):
        raise ValueError("sample_weight must be [rows], finite and >= 0")
    tp, fp, tn, fn = weighted_confusion(p, lab, w)
    ok = (lab != 0) == (p > np.float32(0.5))
    ws = float(np.sum(w.astype(np.float64)))
    r.update(loss=float(np.sum((w * keras_eval.logit_bce_f32(logits, lab)).astype(np.float64)) / p.shape[0]),
             accuracy=float(np.sum(w.astype(np.float64)[ok])) / ws if ws else 0.0,
             roc_auc=keras_eval.roc_auc_from_counts(tp, fp, tn, fn),
             pr_auc=keras_eval.pr_auc_from_counts(tp, fp, tn, fn), tp=tp, fp=fp, tn=tn, fn=fn)
    return r


def fit(model, W, data, label, orders, batch_size: int, dtype=np.float32, hp=None, weights=None):
    """The model oracle's `fit` over the rows in `orders` [epochs][n], batches of `batch_size` consecutive entries,
    the last one partial, with the dataset's row weights `weights` [n] (None: unweighted).  `data`: (movieId,
    userId) for NeuralCF and two towers, the oracle's Rows for the others.  Returns (weights at `dtype`, history:
    per epoch the weighted `keras_evaluate` of the steps' outputs before their updates)."""
    mod = ORACLE[model]
    W = ncf_train.as_dtype(W, dtype)
    opt = mod.Adam(W, dtype, hp)
    label = np.asarray(label)
    ids_only = model in ("neuralcf", "twotowers")
    if model == "widendeep":
        data.bucket(widendeep_train.cross_buckets(W))          # once for all the rows, as its fit does
    history = []
    for order in orders:
        ps, zs, ys, ws = [], [], [], []
        for lo in range(0, len(order), batch_size):
            rows = np.asarray(order[lo:lo + batch_size])
            y = label[rows]
            wb = None if weights is None else np.asarray(weights)[rows]
            if ids_only:
                mid, uid = np.asarray(data[0])[rows], np.asarray(data[1])[rows]
                g, p, z = gradients(model, W, mid, uid, y, dtype, weight=wb)
                opt.step(W, g, {"movieId_embedding": mid, "userId_embedding": uid})
            else:
                r = data.take(rows)
                g, p, z = gradients(model, W, r, y, dtype, weight=wb)
                opt.step(W, g, mod.table_rows(r))
            ps.append(p); zs.append(z); ys.append(y); ws.append(wb)
        res = keras_evaluate(np.concatenate(ps).astype(np.float32), np.concatenate(zs).astype(np.float32),
                             np.concatenate(ys), None if weights is None else np.concatenate(ws))
        history.append({k: res[k] for k in ("loss", "accuracy", "roc_auc", "pr_auc")})
    return W, history
