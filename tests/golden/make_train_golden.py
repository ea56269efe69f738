"""Regenerate the known answers of `tfrecmodel.neuralcf.fit` from the reference checkout.

Run on a machine that has the reference (the GPU machines do not):

    python tests/golden/make_train_golden.py            # about 2-3 minutes per seed, seeds run in parallel

Writes, next to this file:

* `neuralcf_trainset.npz` - `movieId`, `userId`, `label` (int32) of all 88 827 rows of the reference's
  `webroot/sampledata/trainingSamples.csv` in file order: the data NeuralCF.py:77-91 trains on.
* `neuralcf_fit.json` - for each seed S in SEEDS, the float32 oracle (`oracle.ncf_train.fit`) of the script's run:
  the untrained weights `init_weights(default_spec("neuralcf"), S, for_test=False)`, the row order
  `epoch_orders(88827, 5, S)`, batch 12, 5 epochs.  Per seed: the 5-epoch history and
  `oracle.keras_eval.keras_evaluate` of the trained weights on `neuralcf_002_testset.npz` (the 22 440 rows of
  `testSamples.csv`).  `band` holds, per test metric, the seed-to-seed min and max.

`python tests/golden/make_train_golden.py --check` rebuilds the trainset only and compares it with the committed
file (the fast part; the histories are checked by rerunning this script).
"""
import json
import os
import sys
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
    full = features.load_samples_csv(REF)
    return {k: np.ascontiguousarray(full[k], np.int32) for k in ("movieId", "userId", "label")}


def testset():
    z = np.load(os.path.join(HERE, "neuralcf_002_testset.npz"))
    return z["movieId"], z["userId"], z["label"]


def run_seed(seed):
    from oracle import keras_eval, ncf_train
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    z = np.load(os.path.join(HERE, "neuralcf_trainset.npz"))
    W0 = init_weights(default_spec("neuralcf"), seed, for_test=False)
    orders = ncf_train.epoch_orders(len(z["label"]), EPOCHS, seed)
    W, hist, _, opt = ncf_train.fit(W0, z["movieId"], z["userId"], z["label"], orders, BATCH, np.float32)
    tm, tu, tl = testset()
    p, zz, _ = ncf_train.forward(W, tm, tu, np.float32)
    r = keras_eval.keras_evaluate(p, zz, tl)
    return {"seed": seed, "iterations": opt.iterations, "history": hist, "test": {k: r[k] for k in METRICS}}


def main():
    ts = trainset()
    path = os.path.join(HERE, "neuralcf_trainset.npz")
    if "--check" in sys.argv:
        old = np.load(path)
        assert all(np.array_equal(old[k], ts[k]) for k in ts), "trainset differs from the committed file"
        print("trainset matches")
        return
    np.savez_compressed(path, **ts)
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    with Pool(len(SEEDS)) as pool:
        runs = pool.map(run_seed, SEEDS)
    band = {k: [min(r["test"][k] for r in runs), max(r["test"][k] for r in runs)] for k in METRICS}
    res = {"rows": int(len(ts["label"])), "epochs": EPOCHS, "batch_size": BATCH, "seeds": list(SEEDS),
           "runs": runs, "band": band}
    with open(os.path.join(HERE, "neuralcf_fit.json"), "w") as f:
        json.dump(res, f, indent=1)
    for r in runs:
        print(r["seed"], r["test"])
    print("band", band)


if __name__ == "__main__":
    main()
