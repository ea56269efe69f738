"""Regenerate the known answers of `tfrecmodel.widendeep.fit` from the reference checkout.

Run on a machine that has the reference (the GPU machines do not):

    python tests/golden/make_widendeep_train_golden.py     # several minutes per seed, seeds run in parallel

Writes, next to this file:

* `widendeep_samples.npz` - the Wide&Deep columns that `deepfm_trainset.npz` (the 88 827 rows of the reference's
  `trainingSamples.csv`) and `dien_testset.npz` (the 22 440 rows of `testSamples.csv`) lack, row-aligned with
  them, both in file order: `train_movieGenre2` .. `train_movieGenre3`, `train_userGenre2` .. `train_userGenre5`
  as int8 vocabulary indices (-1 = missing) and `train_userRatedMovie1` (int32), and `test_movieGenre2` ..
  `test_userGenre5` (the test file already carries userRatedMovie1).  The script asserts the alignment on
  movieId, userId and label.
* `widendeep_fit.json` - for each seed S in SEEDS, the float32 oracle (`oracle.widendeep_train.fit`) of the
  script's run: the untrained weights `init_weights(default_spec("widendeep"), S, for_test=False)`, the row order
  `epoch_orders(88827, 5, S)`, batch 12, 5 epochs.  Per seed: the 5-epoch history, the oracle's host seconds and
  `oracle.keras_eval.keras_evaluate` of the trained weights on the 22 440 test rows.  `band` holds, per test
  metric, the seed-to-seed min and max.

`python tests/golden/make_widendeep_train_golden.py --check` rebuilds the columns only and compares them with the
committed file (the fast part; the histories are checked by rerunning this script).
"""
import json
import os
import sys
import time
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

DATA = "/root/reference/src/main/resources/webroot/sampledata/"
SEEDS = (0, 1, 2, 3)
EPOCHS, BATCH = 5, 12
METRICS = ("loss", "accuracy", "roc_auc", "pr_auc")
GENRES = ("movieGenre2", "movieGenre3", "userGenre2", "userGenre3", "userGenre4", "userGenre5")


def columns():
    from sparrowrecsys_b200 import features
    out = {}
    for part, csv, base in (("train", "trainingSamples.csv", "deepfm_trainset.npz"),
                            ("test", "testSamples.csv", "dien_testset.npz")):
        full = features.load_samples_csv(os.path.join(DATA, csv))
        have = np.load(os.path.join(HERE, base))
        for k in ("movieId", "userId", "label"):
            assert np.array_equal(np.asarray(full[k], np.int64), have[k].astype(np.int64)), (part, k)
        for k in GENRES:
            out["%s_%s" % (part, k)] = features.genre_to_index(full[k]).astype(np.int8)
        if part == "train":
            out["train_userRatedMovie1"] = np.ascontiguousarray(full["userRatedMovie1"], np.int32)
        else:
            assert np.array_equal(np.asarray(full["userRatedMovie1"], np.int64),
                                  have["userRatedMovie1"].astype(np.int64))
    return out


def load(part):
    """The Wide&Deep feature dict of the train or test rows, from the committed fixtures."""
    base = dict(np.load(os.path.join(HERE, "deepfm_trainset.npz" if part == "train" else "dien_testset.npz")))
    extra = np.load(os.path.join(HERE, "widendeep_samples.npz"))
    for k in extra.files:
        if k.startswith(part + "_"):
            base[k[len(part) + 1:]] = extra[k]
    return base


def run_seed(seed):
    from oracle import keras_eval, widendeep_train
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    t0 = time.time()
    z = load("train")
    W0 = init_weights(default_spec("widendeep"), seed, for_test=False)
    orders = widendeep_train.epoch_orders(len(z["label"]), EPOCHS, seed)
    W, hist, _, opt = widendeep_train.fit(W0, widendeep_train.Rows.from_features(z), z["label"], orders, BATCH,
                                          np.float32)
    seconds = time.time() - t0
    test = load("test")
    p, zz, _ = widendeep_train.forward(W, widendeep_train.Rows.from_features(test), np.float32)
    r = keras_eval.keras_evaluate(p, zz, test["label"])
    return {"seed": seed, "iterations": opt.iterations, "oracle_seconds": round(seconds, 1),
            "history": hist, "test": {k: r[k] for k in METRICS}}


def main():
    cols = columns()
    path = os.path.join(HERE, "widendeep_samples.npz")
    if "--check" in sys.argv:
        old = np.load(path)
        assert sorted(old.files) == sorted(cols), "columns differ from the committed file"
        assert all(old[k].dtype == cols[k].dtype and np.array_equal(old[k], cols[k]) for k in cols), \
            "columns differ from the committed file"
        print("widendeep samples match")
        return
    np.savez_compressed(path, **cols)
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    with Pool(len(SEEDS)) as pool:
        runs = pool.map(run_seed, SEEDS)
    band = {k: [min(r["test"][k] for r in runs), max(r["test"][k] for r in runs)] for k in METRICS}
    res = {"rows": int(len(cols["train_userRatedMovie1"])), "test_rows": int(len(cols["test_movieGenre2"])),
           "epochs": EPOCHS, "batch_size": BATCH, "seeds": list(SEEDS), "runs": runs, "band": band}
    with open(os.path.join(HERE, "widendeep_fit.json"), "w") as f:
        json.dump(res, f, indent=1)
    for r in runs:
        print(r["seed"], r["oracle_seconds"], r["test"])
    print("band", band)


if __name__ == "__main__":
    main()
