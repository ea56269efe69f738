"""Regenerate the known answer of `model.evaluate` from the reference checkout.

Run on a machine that has the reference (the GPU machines do not):

    python tests/golden/make_eval_golden.py

Writes, next to this file:

* `neuralcf_002_testset.npz` - everything `tfrecmodel.neuralcf.evaluate` needs for the whole
  `testSamples.csv` of the reference (`webroot/sampledata/`): `movieId`, `userId`, `label` of all 22 440
  rows in file order; the shipped `modeldata/neuralcf/002` weights, read with `sparrowrecsys_b200.bundle`,
  with the 30001-row user table cut to the users that occur (`user_ids`, `user_rows`; the other rows are
  never read).  The script asserts that the cut table gives the same probabilities as the full one.
* `neuralcf_002_eval.json` - `oracle.keras_eval.keras_evaluate` on the oracle's float32 forward of those
  rows: the four metrics, the confusion counts, the exact rank (Mann-Whitney) ROC AUC beside the
  200-threshold one, and `near`: the rows whose probability lies within 2e-5 of a threshold or of 0.5 -
  the rows a GPU-vs-oracle difference in the last bits could move to another bin or another side.
  Its accuracy equals `full_file_stats.json`'s (asserted).
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from sparrowrecsys_b200 import bundle, features                      # noqa: E402
from sparrowrecsys_b200.spec import default_spec                      # noqa: E402
from oracle import ctr_oracle, keras_eval                            # noqa: E402

REF = "/root/reference/src/main/resources/webroot/"
NEAR = 2e-5


def rank_auc(p, lab):
    """Exact ROC AUC: Mann-Whitney U with tied scores at their average rank."""
    order = np.argsort(p, kind="mergesort")
    ranks = np.empty(len(p))
    ranks[order] = np.arange(1, len(p) + 1)
    _, inv, cnt = np.unique(p, return_inverse=True, return_counts=True)
    ranks = (np.bincount(inv, weights=ranks) / cnt)[inv]
    npos = int((lab == 1).sum())
    nneg = len(lab) - npos
    return float((ranks[lab == 1].sum() - npos * (npos + 1) / 2) / (npos * nneg))


def main():
    full = features.load_samples_csv(REF + "sampledata/testSamples.csv")
    W = bundle.load_neuralcf(REF + "modeldata/neuralcf/002")
    spec = default_spec("neuralcf")
    movie, user, lab = full["movieId"], full["userId"], full["label"]
    feats = {"movieId": movie, "userId": user}
    users = np.unique(user)
    out = {k.replace("/", "__"): v for k, v in W.items() if k != "userId_embedding"}
    out.update(movieId=movie.astype(np.int32), userId=user.astype(np.int32), label=lab.astype(np.int32),
               user_ids=users.astype(np.int32), user_rows=W["userId_embedding"][users])
    np.savez_compressed(os.path.join(HERE, "neuralcf_002_testset.npz"), **out)

    p, z = ctr_oracle.forward(spec, W, feats)
    cut = dict(W)
    cut["userId_embedding"] = np.zeros_like(W["userId_embedding"])
    cut["userId_embedding"][users] = W["userId_embedding"][users]
    p_cut, z_cut = ctr_oracle.forward(spec, cut, feats)
    assert np.array_equal(p, p_cut) and np.array_equal(z, z_cut)

    p, z = p[:, 0], z[:, 0]
    r = keras_eval.keras_evaluate(p, z, lab)
    with open(os.path.join(HERE, "full_file_stats.json")) as f:
        stats = json.load(f)
    assert r["rows"] == stats["rows"] and r["accuracy"] == stats["accuracy"], (r["accuracy"], stats)
    marks = np.concatenate([keras_eval.keras_thresholds().astype(np.float64), [0.5]])
    near = int((np.abs(p.astype(np.float64)[:, None] - marks[None, :]).min(1) <= NEAR).sum())
    res = {"rows": r["rows"], "positives": r["positives"], "correct": r["correct"],
           "loss": r["loss"], "accuracy": r["accuracy"], "roc_auc": r["roc_auc"], "pr_auc": r["pr_auc"],
           "exact_rank_roc_auc": rank_auc(p, lab), "near_tolerance": NEAR, "near": near,
           "tp": r["tp"].tolist(), "fp": r["fp"].tolist(), "tn": r["tn"].tolist(), "fn": r["fn"].tolist()}
    with open(os.path.join(HERE, "neuralcf_002_eval.json"), "w") as f:
        json.dump(res, f, indent=1)
    print({k: v for k, v in res.items() if k not in ("tp", "fp", "tn", "fn")})


if __name__ == "__main__":
    main()
