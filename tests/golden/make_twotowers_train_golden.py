"""Regenerate the known answers of training the two-tower model (neural_cf_model_2) with `training.Trainer`.

    python tests/golden/make_twotowers_train_golden.py      # a few minutes per seed, seeds run in parallel

Reads only committed fixtures (`neuralcf_trainset.npz`, `neuralcf_002_testset.npz`), so it runs without the
reference checkout.  Writes `twotowers_fit.json` next to this file: for each seed S in SEEDS, the float32 oracle
(`oracle.twotowers_train.fit`) of NeuralCF.py's second model trained as the script trains its first -
`neural_cf_model_2` with the script's `hidden_units` [10, 10], E = 10 and the final Dense, from the untrained
weights `init_weights(default_spec("twotowers", hidden=(10, 10)), S, for_test=False)`, the row order
`epoch_orders(88827, 5, S)`, batch 12, 5 epochs over the 88 827 rows of trainingSamples.csv.  Per seed: the
5-epoch history and `oracle.keras_eval.keras_evaluate` of the trained weights on the 22 440 rows of testSamples.csv.
`band` holds, per test metric, the seed-to-seed min and max.
"""
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

SEEDS = (0, 1, 2, 3)
EPOCHS, BATCH = 5, 12
HIDDEN = (10, 10)
METRICS = ("loss", "accuracy", "roc_auc", "pr_auc")


def spec():
    from sparrowrecsys_b200.spec import default_spec
    return default_spec("twotowers", hidden=HIDDEN, final_dense=True)


def run_seed(seed):
    from oracle import keras_eval, twotowers_train
    from sparrowrecsys_b200.training import epoch_orders
    from sparrowrecsys_b200.weights import init_weights
    z = np.load(os.path.join(HERE, "neuralcf_trainset.npz"))
    W0 = init_weights(spec(), seed, for_test=False)
    orders = epoch_orders(len(z["label"]), EPOCHS, seed)
    W, hist, _, opt = twotowers_train.fit(W0, z["movieId"], z["userId"], z["label"], orders, BATCH, np.float32)
    t = np.load(os.path.join(HERE, "neuralcf_002_testset.npz"))
    p, zz, _ = twotowers_train.forward(W, t["movieId"], t["userId"], np.float32)
    r = keras_eval.keras_evaluate(p, zz, t["label"])
    return {"seed": seed, "iterations": opt.iterations, "history": hist, "test": {k: r[k] for k in METRICS}}


def main():
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    rows = int(len(np.load(os.path.join(HERE, "neuralcf_trainset.npz"))["label"]))
    with Pool(len(SEEDS)) as pool:
        runs = pool.map(run_seed, SEEDS)
    band = {k: [min(r["test"][k] for r in runs), max(r["test"][k] for r in runs)] for k in METRICS}
    res = {"model": "twotowers", "emb_dim": spec().emb_dim, "hidden": list(HIDDEN), "final_dense": True,
           "rows": rows, "epochs": EPOCHS, "batch_size": BATCH, "seeds": list(SEEDS), "runs": runs, "band": band}
    with open(os.path.join(HERE, "twotowers_fit.json"), "w") as f:
        json.dump(res, f, indent=1)
    for r in runs:
        print(r["seed"], r["test"])
    print("band", band)


if __name__ == "__main__":
    main()
