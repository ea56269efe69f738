"""CPU oracle of Keras's `model.evaluate` metrics for the reference's CTR models.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

Every CTR script of the reference compiles its model as
`compile(loss='binary_crossentropy', optimizer='adam', metrics=['accuracy', AUC(curve='ROC'),
AUC(curve='PR')])` and ends with `model.evaluate(test_dataset)` (e.g. DIN.py:171-185,
EmbeddingMLP.py:80-91, NeuralCF.py:77-88).  This restates what that call reports under TF 2.0 (the
version that wrote the shipped exports).  TensorFlow is not installable here, so like the rest of the
oracle the restatement is unpinned.  It lives in its own module beside ctr_oracle.py.
"""
from __future__ import annotations

import numpy as np

NUM_THRESHOLDS = 200


def keras_thresholds() -> np.ndarray:
    """`[0.0 - 1e-7] + [(i + 1) * 1.0 / 199 for i in range(198)] + [1.0 + 1e-7]` built in double, each value
    cast to float32 (keras.utils.metrics_utils / AUC.__init__, num_thresholds=200)."""
    kepsilon = 1e-7
    t = [0.0 - kepsilon] + [(i + 1) * 1.0 / (NUM_THRESHOLDS - 1) for i in range(NUM_THRESHOLDS - 2)] \
        + [1.0 + kepsilon]
    return np.array(t, np.float64).astype(np.float32)


def _div_no_nan(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    out = np.zeros(np.broadcast(a, b).shape)
    nz = b != 0
    np.divide(a, b, out=out, where=nz)
    return out


def confusion_counts(probs, labels):
    """(tp, fp, tn, fn), int64 [200] each, by the literal broadcast comparison Keras makes:
    row predicted positive at threshold t when float32(p) > t (strictly); label positive when nonzero."""
    p = np.asarray(probs, np.float32).reshape(-1)
    pos = np.asarray(labels).reshape(-1) != 0
    t = keras_thresholds()
    tp = np.zeros(NUM_THRESHOLDS, np.int64)
    fp = np.zeros(NUM_THRESHOLDS, np.int64)
    for lo in range(0, p.shape[0], 1 << 16):
        pred = p[lo:lo + (1 << 16), None] > t[None, :]        # [rows, 200]
        ps = pos[lo:lo + (1 << 16), None]
        tp += (pred & ps).sum(0)
        fp += (pred & ~ps).sum(0)
    return tp, fp, int((~pos).sum()) - fp, int(pos.sum()) - tp


def roc_auc_from_counts(tp, fp, tn, fn) -> float:
    """AUC(curve='ROC', summation_method='interpolation'): recall = div_no_nan(tp, tp + fn),
    fpr = div_no_nan(fp, fp + tn), sum of (x[:-1] - x[1:]) * (y[:-1] + y[1:]) / 2 with x = fpr, y = recall.
    A single-class input gives 0.0."""
    tp, fp, tn, fn = (np.asarray(v, np.float64) for v in (tp, fp, tn, fn))
    y = _div_no_nan(tp, tp + fn)
    x = _div_no_nan(fp, fp + tn)
    return float(np.sum((x[:-1] - x[1:]) * ((y[:-1] + y[1:]) / 2.0)))


def pr_auc_from_counts(tp, fp, tn, fn) -> float:
    """AUC(curve='PR', summation_method='interpolation') = Keras's interpolate_pr_auc (Davis & Goadrich 2006),
    line by line:
        dtp = tp[:-1] - tp[1:];  p = tp + fp;  dp = p[:-1] - p[1:]
        slope = div_no_nan(dtp, max(dp, 0));  intercept = tp[1:] - slope * p[1:]
        ratio = where(p[:-1] > 0 & p[1:] > 0, div_no_nan(p[:-1], max(p[1:], 0)), 1)
        sum(div_no_nan(slope * (dtp + intercept * log(ratio)), max(tp[1:] + fn[1:], 0)))"""
    tp, fp, tn, fn = (np.asarray(v, np.float64) for v in (tp, fp, tn, fn))
    dtp = tp[:-1] - tp[1:]
    p = tp + fp
    dp = p[:-1] - p[1:]
    slope = _div_no_nan(dtp, np.maximum(dp, 0.0))
    intercept = tp[1:] - slope * p[1:]
    both = (p[:-1] > 0) & (p[1:] > 0)
    ratio = np.where(both, _div_no_nan(p[:-1], np.maximum(p[1:], 0.0)), 1.0)
    with np.errstate(divide="ignore"):
        logr = np.log(ratio)
    return float(np.sum(_div_no_nan(slope * (dtp + intercept * logr), np.maximum(tp[1:] + fn[1:], 0.0))))


def logit_bce_f32(logits, labels) -> np.ndarray:
    """Per-row binary_crossentropy of a sigmoid output layer, float32 as TF computes it: Keras sees the
    `Sigmoid` op and takes sigmoid_cross_entropy_with_logits on its input,
    max(x, 0) - x*z + log1p(exp(-|x|)), instead of the clipped-probability formula (a logit of 30 with
    label 0 costs about 30, not 16.118)."""
    x = np.asarray(logits, np.float32).reshape(-1)
    z = (np.asarray(labels).reshape(-1) != 0).astype(np.float32)
    return (np.maximum(x, np.float32(0)) - x * z) + np.log1p(np.exp(-np.abs(x)))


def clipped_bce(probs, labels) -> np.ndarray:
    """The formula Keras does NOT take for a sigmoid output (kept for tests that tell the two apart):
    -(z log(p') + (1 - z) log(1 - p')), p' = clip(p, 1e-7, 1 - 1e-7)."""
    p = np.clip(np.asarray(probs, np.float64).reshape(-1), 1e-7, 1 - 1e-7)
    z = (np.asarray(labels).reshape(-1) != 0).astype(np.float64)
    return -(z * np.log(p) + (1 - z) * np.log(1 - p))


def keras_evaluate(probs, logits, labels) -> dict:
    """What `model.evaluate` reports for the reference's compile line, in float64 on top of the float32
    per-row terms.

    * Thresholds: `keras_thresholds()`, 200 float32 values.
    * Confusion counts: at threshold t a row is predicted positive when float32(p) > t, strictly; a label is
      positive when nonzero.  TP, FP, TN, FN are exact integers here; Keras keeps them in float32 variables,
      which stop being exact above 2^24 rows - a difference kept on purpose.
    * roc_auc / pr_auc: `roc_auc_from_counts` / `pr_auc_from_counts` (0.0 for a single class).
    * accuracy: binary_accuracy, correct when label == (p > 0.5); p == 0.5 is a negative prediction.
    * loss: the row mean of `logit_bce_f32` (float32 per row, as TF).  The row mean is Keras's
      batch-weighted mean; TF 2.0 may average batch means without weights, which is the same value when
      every batch is full (batch 12 over the 22 440 test rows is exactly 1870 batches).
    * errors: Keras asserts 0 <= y_pred <= 1, so a NaN or out-of-range probability raises ValueError; so does
      a label other than 0 and 1 (the reference feeds only 0/1; its accuracy and AUC disagree on others).

    Returns loss, accuracy, roc_auc, pr_auc, rows, positives, correct, tp, fp, tn, fn."""
    p = np.asarray(probs, np.float32).reshape(-1)
    lab = np.asarray(labels).reshape(-1)
    if p.shape[0] != lab.shape[0] or p.shape[0] != np.asarray(logits).reshape(-1).shape[0]:
        raise ValueError("probs, logits and labels differ in length")
    if p.shape[0] == 0:
        raise ValueError("no rows")
    if not np.all((p >= 0) & (p <= 1)):
        raise ValueError("a probability is NaN or outside [0, 1]")
    if not np.all((lab == 0) | (lab == 1)):
        raise ValueError("labels must be 0 or 1")
    tp, fp, tn, fn = confusion_counts(p, lab)
    pos = lab != 0
    correct = int((pos == (p > np.float32(0.5))).sum())
    loss = float(np.sum(logit_bce_f32(logits, lab).astype(np.float64)) / p.shape[0])
    return {"loss": loss, "accuracy": correct / p.shape[0], "roc_auc": roc_auc_from_counts(tp, fp, tn, fn),
            "pr_auc": pr_auc_from_counts(tp, fp, tn, fn), "rows": int(p.shape[0]), "positives": int(pos.sum()),
            "correct": correct, "tp": tp, "fp": fp, "tn": tn, "fn": fn}
