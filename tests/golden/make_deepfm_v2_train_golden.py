"""Regenerate the known answers of `tfrecmodel.deepfm_v2.fit` from the committed sample fixtures.

    python tests/golden/make_deepfm_v2_train_golden.py     # several minutes per seed, seeds run in parallel

DeepFM_v2 reads exactly the columns of `deepfm_trainset.npz` (the 88 827 rows of the reference's
`trainingSamples.csv`) and `dien_testset.npz` (the 22 440 rows of `testSamples.csv`), so no new sample file is
needed.  Writes `deepfm_v2_fit.json` next to this file: for each seed S in SEEDS, the float32 oracle
(`oracle.deepfm_v2_train.fit`) of the script's run - the untrained weights
`init_weights(default_spec("deepfm_v2"), S, for_test=False)`, the row order `epoch_orders(88827, 5, S)`, batch 12,
5 epochs.  Per seed: the 5-epoch history, the oracle's host seconds and `oracle.keras_eval.keras_evaluate` of the
trained weights on the 22 440 test rows.  `band` holds, per test metric, the seed-to-seed min and max.
"""
import json
import os
import sys
import time
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

SEEDS = (0, 1, 2, 3)
EPOCHS, BATCH = 5, 12
METRICS = ("loss", "accuracy", "roc_auc", "pr_auc")


def load(part):
    """The DeepFM_v2 feature dict of the train or test rows, from the committed fixtures."""
    return dict(np.load(os.path.join(HERE, "deepfm_trainset.npz" if part == "train" else "dien_testset.npz")))


def run_seed(seed):
    from oracle import deepfm_v2_train, keras_eval
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    t0 = time.time()
    z = load("train")
    W0 = init_weights(default_spec("deepfm_v2"), seed, for_test=False)
    orders = deepfm_v2_train.epoch_orders(len(z["label"]), EPOCHS, seed)
    W, hist, _, opt = deepfm_v2_train.fit(W0, deepfm_v2_train.Rows.from_features(z), z["label"], orders, BATCH,
                                          np.float32)
    seconds = time.time() - t0
    test = load("test")
    p, zz, _ = deepfm_v2_train.forward(W, deepfm_v2_train.Rows.from_features(test), np.float32)
    r = keras_eval.keras_evaluate(p, zz, test["label"])
    return {"seed": seed, "iterations": opt.iterations, "oracle_seconds": round(seconds, 1),
            "history": hist, "test": {k: r[k] for k in METRICS}}


def main():
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    with Pool(len(SEEDS)) as pool:
        runs = pool.map(run_seed, SEEDS)
    band = {k: [min(r["test"][k] for r in runs), max(r["test"][k] for r in runs)] for k in METRICS}
    res = {"rows": int(len(load("train")["label"])), "test_rows": int(len(load("test")["label"])),
           "epochs": EPOCHS, "batch_size": BATCH, "seeds": list(SEEDS), "runs": runs, "band": band}
    with open(os.path.join(HERE, "deepfm_v2_fit.json"), "w") as f:
        json.dump(res, f, indent=1)
    for r in runs:
        print(r["seed"], r["oracle_seconds"], r["test"])
    print("band", band)


if __name__ == "__main__":
    main()
