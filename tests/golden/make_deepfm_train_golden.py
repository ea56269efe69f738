"""Regenerate the known answers of `tfrecmodel.deepfm.fit` from the reference checkout.

Run on a machine that has the reference (the GPU machines do not):

    python tests/golden/make_deepfm_train_golden.py     # several minutes per seed, seeds run in parallel

Writes, next to this file:

* `deepfm_trainset.npz` - the 88 827 rows of the reference's `webroot/sampledata/trainingSamples.csv` in file
  order, with the columns DeepFM.py's model reads: `movieId`, `userId`, `label` (int32), the 7 numerics as
  `features.load_samples_csv` types them, and `movieGenre1` / `userGenre1` as int8 vocabulary indices (-1 =
  missing), as `dien_testset.npz` stores them.
* `deepfm_fit.json` - for each seed S in SEEDS, the float32 oracle (`oracle.deepfm_train.fit`) of the script's
  run: the untrained weights `init_weights(default_spec("deepfm"), S, for_test=False)`, the row order
  `epoch_orders(88827, 5, S)`, batch 12, 5 epochs.  Per seed: the 5-epoch history and
  `oracle.keras_eval.keras_evaluate` of the trained weights on `dien_testset.npz` (the 22 440 rows of
  `testSamples.csv`, which carry every DeepFM column).  `band` holds, per test metric, the seed-to-seed min and max.

`python tests/golden/make_deepfm_train_golden.py --check` rebuilds the trainset only and compares it with the
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

REF = "/root/reference/src/main/resources/webroot/sampledata/trainingSamples.csv"
SEEDS = (0, 1, 2, 3)
EPOCHS, BATCH = 5, 12
METRICS = ("loss", "accuracy", "roc_auc", "pr_auc")


def trainset():
    from sparrowrecsys_b200 import features
    from sparrowrecsys_b200.spec import NUMERIC_KEYS
    full = features.load_samples_csv(REF)
    out = {k: np.ascontiguousarray(full[k], np.int32) for k in ("movieId", "userId", "label")}
    for k in NUMERIC_KEYS:
        out[k] = np.ascontiguousarray(full[k])
    for k in ("movieGenre1", "userGenre1"):
        out[k] = features.genre_to_index(full[k]).astype(np.int8)
    return out


def run_seed(seed):
    from oracle import deepfm_train, keras_eval
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    t0 = time.time()
    z = dict(np.load(os.path.join(HERE, "deepfm_trainset.npz")))
    W0 = init_weights(default_spec("deepfm"), seed, for_test=False)
    orders = deepfm_train.epoch_orders(len(z["label"]), EPOCHS, seed)
    W, hist, _, opt = deepfm_train.fit(W0, deepfm_train.Rows.from_features(z), z["label"], orders, BATCH,
                                       np.float32)
    test = dict(np.load(os.path.join(HERE, "dien_testset.npz")))
    p, zz, _ = deepfm_train.forward(W, deepfm_train.Rows.from_features(test), np.float32)
    r = keras_eval.keras_evaluate(p, zz, test["label"])
    return {"seed": seed, "iterations": opt.iterations, "oracle_seconds": round(time.time() - t0, 1),
            "history": hist, "test": {k: r[k] for k in METRICS}}


def main():
    ts = trainset()
    path = os.path.join(HERE, "deepfm_trainset.npz")
    if "--check" in sys.argv:
        old = np.load(path)
        assert sorted(old.files) == sorted(ts), "trainset columns differ from the committed file"
        assert all(old[k].dtype == ts[k].dtype and np.array_equal(old[k], ts[k]) for k in ts), \
            "trainset differs from the committed file"
        print("trainset matches")
        return
    np.savez_compressed(path, **ts)
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    with Pool(len(SEEDS)) as pool:
        runs = pool.map(run_seed, SEEDS)
    band = {k: [min(r["test"][k] for r in runs), max(r["test"][k] for r in runs)] for k in METRICS}
    res = {"rows": int(len(ts["label"])), "epochs": EPOCHS, "batch_size": BATCH, "seeds": list(SEEDS),
           "runs": runs, "band": band}
    with open(os.path.join(HERE, "deepfm_fit.json"), "w") as f:
        json.dump(res, f, indent=1)
    for r in runs:
        print(r["seed"], r["oracle_seconds"], r["test"])
    print("band", band)


if __name__ == "__main__":
    main()
