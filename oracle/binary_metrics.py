"""mllib's `BinaryClassificationMetrics` (Spark 2.4.3, the reference's pom.xml) in numpy float64: what
`OFF/evaluate/Evaluator.scala` prints, and what ml's `BinaryClassificationEvaluator` returns.

The rules below are restated from memory of Spark's source (`BinaryClassificationMetrics`,
`BinaryLabelCounter`, `BinaryConfusionMatrixImpl`, the `BinaryClassificationMetricComputer`s and
`AreaUnderCurve`); no artefact of Spark pins them.  Each rule lives in one named function, so that a
correction is one edit:

* `is_positive`          BinaryLabelCounter: a label > 0.5 is a positive, anything else (NaN too) a negative.
* `descending_key`       combineByKey's boxed Double equality and sortByKey(ascending = false)'s Double.compare:
                         every NaN is one key and sorts first; 0.0 and -0.0 are two thresholds, 0.0 above.
* `bin_counts`           numBins: grouping = countsSize / numBins; under 2 nothing is merged, else runs of
                         `grouping` consecutive thresholds merge, each taking its first (highest) score and the
                         sum of its counts; the last run may be shorter.  One partition (Spark groups per
                         partition).
* `precision`, `recall`, `false_positive_rate`, `f_measure`   the metric computers.
* `roc_points`, `pr_points`   roc() and pr() with their end points.
* `trapezoid_terms`, `area_under_curve`   AreaUnderCurve.of: the trapezoids summed left to right in double.

Empty input is rejected: Spark's pr() calls first() on an empty RDD.
"""
from __future__ import annotations

import numpy as np

_SIGN = np.uint64(1 << 63)


def is_positive(labels) -> np.ndarray:
    """BinaryLabelCounter.+=: label > 0.5 counts as a positive, everything else - NaN included - as a negative."""
    with np.errstate(invalid="ignore"):
        return np.asarray(labels, np.float64) > 0.5


def descending_key(scores) -> np.ndarray:
    """The uint64 whose ascending order is Spark's threshold order and whose equality is its grouping: combineByKey
    compares boxed Doubles with equals (doubleToLongBits: every NaN one key, -0.0 != 0.0) and sortByKey(false)
    orders by Double.compare descending (NaN first, then +inf, ..., 0.0, -0.0, ..., -inf)."""
    s = np.ascontiguousarray(scores, np.float64)
    b = s.view(np.uint64)
    asc = np.where(b >> np.uint64(63) == 1, ~b, b | _SIGN)
    return np.where(np.isnan(s), np.uint64(0), ~asc)


def key_score(key) -> np.ndarray:
    """The score of a descending key (every NaN comes back as numpy's canonical NaN)."""
    k = np.asarray(key, np.uint64)
    asc = ~k
    b = np.where(asc >> np.uint64(63) == 1, asc & ~_SIGN, ~asc)
    return np.where(k == 0, np.nan, b.view(np.float64))


def group_scores(scores, labels):
    """The distinct scores in threshold order, with the positives and negatives of each."""
    key = descending_key(scores)
    pos = is_positive(labels)
    if key.shape != pos.shape or key.ndim != 1:
        raise ValueError("scores and labels must be 1-D arrays of one length")
    order = np.argsort(key, kind="stable")
    k, p = key[order], pos[order].astype(np.int64)
    starts = np.flatnonzero(np.r_[True, k[1:] != k[:-1]]) if k.size else np.zeros(0, np.int64)
    npos = np.add.reduceat(p, starts) if k.size else np.zeros(0, np.int64)
    cnt = np.diff(np.r_[starts, k.size])
    return key_score(k[starts]), npos.astype(np.int64), (cnt - npos).astype(np.int64)


def bin_counts(thresholds, pos, neg, num_bins: int):
    """The numBins down-sampling of one partition: grouping = countsSize / numBins (integer division); below 2
    nothing is merged; otherwise each run of `grouping` consecutive thresholds becomes one, with the run's first
    (highest) score and the sum of its counts, the last run possibly shorter.  numBins 0 means no binning."""
    if num_bins < 0:
        raise ValueError("numBins must be >= 0, got %d" % num_bins)
    m = len(thresholds)
    grouping = m // num_bins if num_bins > 0 else 0
    if grouping < 2:
        return np.asarray(thresholds), np.asarray(pos), np.asarray(neg)
    starts = np.arange(0, m, grouping)
    return (np.asarray(thresholds)[starts], np.add.reduceat(pos, starts), np.add.reduceat(neg, starts))


def precision(tp, fp) -> np.ndarray:
    """Precision: TP / (TP + FP), 1.0 when nothing is predicted positive."""
    tp, tot = np.asarray(tp, np.int64), np.asarray(tp, np.int64) + np.asarray(fp, np.int64)
    return np.where(tot == 0, 1.0, tp.astype(np.float64) / np.maximum(tot, 1).astype(np.float64))


def recall(tp, positives: int) -> np.ndarray:
    """Recall: TP / P, 0.0 when there is no positive."""
    tp = np.asarray(tp, np.int64).astype(np.float64)
    return np.zeros_like(tp) if positives == 0 else tp / float(positives)


def false_positive_rate(fp, negatives: int) -> np.ndarray:
    """FalsePositiveRate: FP / N, 0.0 when there is no negative."""
    fp = np.asarray(fp, np.int64).astype(np.float64)
    return np.zeros_like(fp) if negatives == 0 else fp / float(negatives)


def f_measure(p, r, beta: float) -> np.ndarray:
    """FMeasure(beta): (1 + beta^2) * (p * r / (beta^2 * p + r)), 0.0 when p + r == 0."""
    b2 = float(beta) * float(beta)
    p, r = np.asarray(p, np.float64), np.asarray(r, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        v = (1.0 + b2) * (p * r / (b2 * p + r))
    return np.where(p + r == 0, 0.0, v)


def roc_points(fpr, rec) -> np.ndarray:
    """roc(): (0, 0), (FPR, recall) per threshold, (1, 1)."""
    return np.concatenate([[[0.0, 0.0]], np.stack([fpr, rec], 1), [[1.0, 1.0]]])


def pr_points(rec, prec) -> np.ndarray:
    """pr(): (0, the first threshold's precision), then (recall, precision) per threshold."""
    return np.concatenate([[[0.0, prec[0]]], np.stack([rec, prec], 1)])


def trapezoid_terms(points) -> np.ndarray:
    """AreaUnderCurve.trapezoid of each consecutive pair: (x2 - x1) * (y2 + y1) / 2.0."""
    pt = np.asarray(points, np.float64)
    return (pt[1:, 0] - pt[:-1, 0]) * (pt[1:, 1] + pt[:-1, 1]) / 2.0


def area_under_curve(points) -> float:
    """AreaUnderCurve.of: the trapezoids added left to right in double (one partition)."""
    t = trapezoid_terms(points)
    return float(np.cumsum(t)[-1]) if t.size else 0.0


class BinaryMetrics:
    """BinaryClassificationMetrics(scoreAndLabels, numBins) of one score set."""

    def __init__(self, scores, labels, num_bins: int = 0):
        thr, pos, neg = group_scores(scores, labels)
        if thr.size == 0:
            raise ValueError("BinaryClassificationMetrics needs at least one (score, label) pair")
        self._from_counts(thr, pos, neg, num_bins)

    @classmethod
    def from_counts(cls, thresholds, pos, neg, num_bins: int = 0):
        """From the distinct scores in threshold order and their counts (what group_scores returns)."""
        self = cls.__new__(cls)
        self._from_counts(np.asarray(thresholds, np.float64), np.asarray(pos, np.int64),
                          np.asarray(neg, np.int64), num_bins)
        return self

    def _from_counts(self, thr, pos, neg, num_bins):
        self.threshold_array, pos, neg = bin_counts(thr, pos, neg, num_bins)
        self.tp, self.fp = np.cumsum(pos, dtype=np.int64), np.cumsum(neg, dtype=np.int64)
        self.positives, self.negatives = int(self.tp[-1]), int(self.fp[-1])
        self.n = self.positives + self.negatives
        self.precision = precision(self.tp, self.fp)
        self.recall = recall(self.tp, self.positives)
        self.fpr = false_positive_rate(self.fp, self.negatives)

    def thresholds(self) -> np.ndarray:
        return self.threshold_array

    def roc(self) -> np.ndarray:
        return roc_points(self.fpr, self.recall)

    def pr(self) -> np.ndarray:
        return pr_points(self.recall, self.precision)

    def area_under_roc(self) -> float:
        return area_under_curve(self.roc())

    def area_under_pr(self) -> float:
        return area_under_curve(self.pr())

    def precision_by_threshold(self) -> np.ndarray:
        return np.stack([self.threshold_array, self.precision], 1)

    def recall_by_threshold(self) -> np.ndarray:
        return np.stack([self.threshold_array, self.recall], 1)

    def f_measure_by_threshold(self, beta: float = 1.0) -> np.ndarray:
        return np.stack([self.threshold_array, f_measure(self.precision, self.recall, beta)], 1)
