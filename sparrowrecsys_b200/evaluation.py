"""Exact binary-classification metrics on the GPU: mllib's `BinaryClassificationMetrics` (Spark 2.4.3).

This is the reference's `OFF/evaluate/Evaluator.scala`: it builds `BinaryClassificationMetrics` over a predictions
frame's `(probability[1], label)` and prints `areaUnderPR` and `areaUnderROC`.  Unlike Keras's 200-threshold AUC
(`CTRModel.evaluate`), every distinct score is a threshold, so the areas are exact.  DESIGN.md section 4.22 gives the
semantics; `oracle/binary_metrics.py` restates them.

* `BinaryClassificationMetrics(scores, labels, num_bins=0, set_offsets=None)` evaluates one or many score sets in
  one device call (`srs_binary_metrics_create_host`, or `_create_device` for torch CUDA tensors) and reads each
  set's curves on request.
* `BinaryClassificationEvaluator(metric_name)` is ml's evaluator ("areaUnderROC" or "areaUnderPR").
* `evaluate(probabilities, labels)` is Evaluator.evaluate: it prints the two lines and returns both areas.

    python -m sparrowrecsys_b200.evaluation predictions.csv
    python -m sparrowrecsys_b200.evaluation --model neuralcf --savedmodel DIR samples.csv
"""
from __future__ import annotations

import ctypes as C
import csv
import math
import sys
from typing import Optional, Sequence, Tuple

import numpy as np

from . import _lib


def _p(a: np.ndarray):
    return a.ctypes.data


class BinaryClassificationMetrics:
    """BinaryClassificationMetrics(scoreAndLabels, numBins) of one or more score sets.

    `scores` and `labels` are 1-D numpy arrays (float64 on the way in; a label > 0.5 is a positive), or torch CUDA
    tensors - float32 scores and integer labels (positive when > 0), as `CTRModel` produces them - which are read
    on their device.  `set_offsets` (int64 [n_sets + 1], 0 .. n, strictly increasing) cuts the pairs into sets that
    are evaluated independently; every method takes the set's index."""

    def __init__(self, scores, labels, num_bins: int = 0, set_offsets: Optional[Sequence[int]] = None,
                 device: int = 0):
        self._h = None
        lib = _lib.load()
        self._lib = lib
        off = None if set_offsets is None else np.ascontiguousarray(set_offsets, np.int64)
        n_sets = 1 if off is None else off.shape[0] - 1
        h = C.c_void_p()
        if hasattr(scores, "is_cuda"):
            import torch
            if not scores.is_cuda or scores.dtype != torch.float32 or scores.dim() != 1:
                raise TypeError("device scores must be a 1-D float32 CUDA tensor")
            if not getattr(labels, "is_cuda", False) or labels.shape != scores.shape \
                    or labels.device != scores.device or labels.is_floating_point():
                raise TypeError("device labels must be an integer CUDA tensor shaped and placed like the scores")
            s, y = scores.contiguous(), labels.to(torch.int32).contiguous()
            self.device = scores.device.index
            stream = torch.cuda.current_stream(scores.device).cuda_stream
            rc = lib.srs_binary_metrics_create_device(s.data_ptr(), y.data_ptr(), s.shape[0],
                                                      None if off is None else _p(off), n_sets, int(num_bins),
                                                      self.device, stream, C.byref(h))
        else:
            s = np.ascontiguousarray(scores, np.float64)
            y = np.ascontiguousarray(labels, np.float64)
            if s.ndim != 1 or s.shape != y.shape:
                raise ValueError("scores and labels must be 1-D arrays of one length")
            self.device = int(device)
            rc = lib.srs_binary_metrics_create_host(_p(s), _p(y), s.shape[0], None if off is None else _p(off),
                                                    n_sets, int(num_bins), self.device, C.byref(h))
        _lib.check(rc)
        self._h = h
        self.n_sets = n_sets

    def close(self):
        if getattr(self, "_h", None):
            self._lib.srs_binary_metrics_destroy(self._h)
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

    def summary(self, set: int = 0) -> _lib.SrsBinarySummary:
        """n, positives, negatives, thresholds (after binning) and both areas of one set."""
        out = _lib.SrsBinarySummary()
        _lib.check(self._lib.srs_binary_metrics_summary(self._h, int(set), C.byref(out)))
        return out

    def _curve(self, set: int, which: int, beta: float = 1.0) -> np.ndarray:
        T = self.summary(set).thresholds
        shape = {_lib.SRS_BM_ROC: (T + 2, 2), _lib.SRS_BM_PR: (T + 1, 2), _lib.SRS_BM_THRESHOLDS: (T,)}.get(
            which, (T, 2))
        out = np.empty(shape, np.float64)
        _lib.check(self._lib.srs_binary_metrics_curve(self._h, int(set), which, float(beta), _p(out)))
        return out

    def area_under_roc(self, set: int = 0) -> float:
        return self.summary(set).area_under_roc

    def area_under_pr(self, set: int = 0) -> float:
        return self.summary(set).area_under_pr

    def roc(self, set: int = 0) -> np.ndarray:
        """[(0, 0), (FPR, recall) per threshold..., (1, 1)] as float64 [T + 2, 2]."""
        return self._curve(set, _lib.SRS_BM_ROC)

    def pr(self, set: int = 0) -> np.ndarray:
        """[(0, the first precision), (recall, precision) per threshold...] as float64 [T + 1, 2]."""
        return self._curve(set, _lib.SRS_BM_PR)

    def thresholds(self, set: int = 0) -> np.ndarray:
        return self._curve(set, _lib.SRS_BM_THRESHOLDS)

    def precision_by_threshold(self, set: int = 0) -> np.ndarray:
        return self._curve(set, _lib.SRS_BM_PRECISION)

    def recall_by_threshold(self, set: int = 0) -> np.ndarray:
        return self._curve(set, _lib.SRS_BM_RECALL)

    def f_measure_by_threshold(self, beta: float = 1.0, set: int = 0) -> np.ndarray:
        return self._curve(set, _lib.SRS_BM_FMEASURE, beta)

    def confusions(self, set: int = 0) -> Tuple[np.ndarray, np.ndarray]:
        """The cumulative true and false positives (int64 [T]) down the thresholds."""
        T = self.summary(set).thresholds
        tp, fp = np.empty(T, np.int64), np.empty(T, np.int64)
        _lib.check(self._lib.srs_binary_metrics_confusion(self._h, int(set), _p(tp), _p(fp)))
        return tp, fp


class BinaryClassificationEvaluator:
    """ml's BinaryClassificationEvaluator (Spark 2.4): the area `metric_name` of BinaryClassificationMetrics at
    numBins 0."""

    METRICS = ("areaUnderROC", "areaUnderPR")

    def __init__(self, metric_name: str = "areaUnderROC"):
        if metric_name not in self.METRICS:
            raise ValueError("metric_name must be one of %s, got %r" % (self.METRICS, metric_name))
        self.metric_name = metric_name

    def evaluate(self, scores, labels) -> float:
        with BinaryClassificationMetrics(scores, labels) as m:
            return m.area_under_roc() if self.metric_name == "areaUnderROC" else m.area_under_pr()


def java_double(x: float) -> str:
    """Java's Double.toString layout, which Scala's string concatenation prints: "NaN", "Infinity", a plain decimal
    with at least one fractional digit for 1e-3 <= |x| < 1e7, otherwise d.ddd"E"exp.  The digits are the shortest
    that read back to x, as Java 19 and later print them.  Spark 2.4.3 runs on Java 8, whose Double.toString now and
    then writes a longer digit string for the same double, so in rare cases a printed line differs from the
    reference's in its last digits while the value is the same."""
    x = float(x)
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "Infinity" if x > 0 else "-Infinity"
    if x == 0 or 1e-3 <= abs(x) < 1e7:
        return repr(x)                     # repr uses no exponent in this range and always writes ".d"
    mant, exp = np.format_float_scientific(x, unique=True, trim="0").split("e")
    return mant + "E" + str(int(exp))


def evaluate(probabilities, labels, device: int = 0) -> Tuple[float, float]:
    """Evaluator.evaluate: BinaryClassificationMetrics over (probability of class 1, label); prints
    "AUC under PR = ..." then "AUC under ROC = ..." and returns (area under PR, area under ROC)."""
    with BinaryClassificationMetrics(probabilities, labels, device=device) as m:
        pr, roc = m.area_under_pr(), m.area_under_roc()
    print("AUC under PR = " + java_double(pr))
    print("AUC under ROC = " + java_double(roc))
    return pr, roc


def read_predictions_csv(path: str) -> Tuple[np.ndarray, np.ndarray]:
    """`label` and `probability` columns of a CSV; a probability written as a vector "[p0,p1]" gives p1 (what
    Evaluator.scala reads), a plain number is taken as p1 itself."""
    with open(path, newline="") as f:
        reader = csv.DictReader(f)
        if not reader.fieldnames or "label" not in reader.fieldnames or "probability" not in reader.fieldnames:
            raise ValueError("%s needs 'label' and 'probability' columns" % path)
        lab, prob = [], []
        for row in reader:
            p = row["probability"].strip()
            prob.append(float(p.strip("[]").split(",")[1]) if p.startswith("[") else float(p))
            lab.append(float(row["label"]))
    return np.array(prob, np.float64), np.array(lab, np.float64)


def main(argv=None) -> int:
    import argparse
    ap = argparse.ArgumentParser(prog="python -m sparrowrecsys_b200.evaluation",
                                 description="Evaluator.scala: exact area under PR and ROC of binary predictions")
    ap.add_argument("csv", help="predictions.csv (label, probability), or with --savedmodel a samples CSV")
    ap.add_argument("--model", default="neuralcf", help="the SavedModel's layout (CTRModel.from_savedmodel)")
    ap.add_argument("--savedmodel", help="score the samples with this export first")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    if a.savedmodel:
        from .features import load_samples_csv
        from .model import CTRModel
        feats = load_samples_csv(a.csv)
        with CTRModel.from_savedmodel(a.savedmodel, model=a.model, device=a.device) as m:
            probs = m.predict(feats)[:, 0].astype(np.float64)
        labels = feats["label"].astype(np.float64)
    else:
        probs, labels = read_predictions_csv(a.csv)
    evaluate(probs, labels, device=a.device)
    return 0


if __name__ == "__main__":
    sys.exit(main())
