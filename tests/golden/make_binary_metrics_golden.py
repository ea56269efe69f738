"""Regenerate the known answer of BinaryClassificationMetrics on the reference's test rows.

    python tests/golden/make_binary_metrics_golden.py

Writes `binary_metrics.json` next to this file: `oracle.binary_metrics` (numBins 0) on the float32 probabilities of
the oracle's forward of `modeldata/neuralcf/002` over the 22 440 rows of `neuralcf_002_testset.npz` - the counts,
both areas, the threshold count, every 500th point of each curve (and the last) - and, beside them, Keras's
200-threshold areas of the same probabilities from `neuralcf_002_eval.json`.  Needs only files under tests/golden.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import binary_metrics as BM, ctr_oracle                    # noqa: E402
from sparrowrecsys_b200.spec import default_spec                        # noqa: E402

STEP = 500


def testset_probabilities():
    """The oracle's float32 probabilities of neuralcf/002 on the test rows, and their labels."""
    z = np.load(os.path.join(HERE, "neuralcf_002_testset.npz"))
    W = {k.replace("__", "/"): z[k] for k in z.files
         if k not in ("user_ids", "user_rows", "movieId", "userId", "label")}
    table = np.zeros((30001, z["user_rows"].shape[1]), np.float32)
    table[z["user_ids"]] = z["user_rows"]
    W["userId_embedding"] = table
    p, _ = ctr_oracle.forward(default_spec("neuralcf"), W, {"movieId": z["movieId"], "userId": z["userId"]})
    return p[:, 0].astype(np.float32), z["label"].astype(np.int32)


def sampled(a):
    idx = sorted(set(range(0, a.shape[0], STEP)) | {a.shape[0] - 1})
    return {"index": idx, "values": a[idx].tolist()}


def main():
    p, y = testset_probabilities()
    m = BM.BinaryMetrics(p.astype(np.float64), y.astype(np.float64))
    with open(os.path.join(HERE, "neuralcf_002_eval.json")) as f:
        keras = json.load(f)
    res = {"rows": m.n, "positives": m.positives, "negatives": m.negatives,
           "thresholds": int(m.thresholds().shape[0]),
           "area_under_roc": m.area_under_roc(), "area_under_pr": m.area_under_pr(),
           "keras_roc_auc": keras["roc_auc"], "keras_pr_auc": keras["pr_auc"],
           "roc": sampled(m.roc()), "pr": sampled(m.pr()), "threshold_values": sampled(m.thresholds()),
           "tp": sampled(m.tp), "fp": sampled(m.fp)}
    with open(os.path.join(HERE, "binary_metrics.json"), "w") as f:
        json.dump(res, f, indent=1)
    print({k: res[k] for k in ("rows", "positives", "thresholds", "area_under_roc", "area_under_pr",
                               "keras_roc_auc", "keras_pr_auc")})
    print("keras - exact: roc %.3e  pr %.3e" % (res["keras_roc_auc"] - res["area_under_roc"],
                                                 res["keras_pr_auc"] - res["area_under_pr"]))


if __name__ == "__main__":
    main()
