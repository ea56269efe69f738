"""Regenerate the known answers of `tfrecmodel.dien.fit` from the reference checkout.

Run on a machine that has the reference (the GPU machines do not):

    python tests/golden/make_dien_train_golden.py     # several minutes per seed, seeds run in parallel

Writes, next to this file:

* `dien_train_samples.npz` - the DIEN columns that `deepfm_trainset.npz` (the 88 827 rows of the reference's
  `trainingSamples.csv`, in file order) and `widendeep_samples.npz` (its `train_userRatedMovie1`) lack:
  `userRatedMovie2` .. `userRatedMovie5` (int32, 0 = padding), row-aligned.  The script asserts the alignment on
  movieId, userId and label.
* `dien_fit.json` - for each seed S in SEEDS, the float32 oracle (`oracle.dien_train.fit`) of DIEN.py's run: the
  untrained weights `init_weights(default_spec("dien"), S, for_test=False)` with `init_aux_weights(spec, S)`, the
  negatives `negative_history(train, 5, seed=2020)` (DIEN.py:49), file order every epoch (the script's dataset has
  no shuffle), batch 12, 5 epochs.  Per seed: the 5-epoch history {loss, auc, auc_value}, the oracle's host
  seconds and `model.evaluate` of the trained weights on the 22 440 test rows in batches of 12 with the negatives
  `negative_history(test, 5, seed=2021)` (DIEN.py:50), as `CTRModel.dien_evaluate` defines it.  `band` holds, per
  test metric, the seed-to-seed min and max.

`python tests/golden/make_dien_train_golden.py --check` rebuilds the columns only and compares them with the
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
EPOCHS, BATCH, T = 5, 12, 5
METRICS = ("loss", "auc", "auc_value")
HIST = tuple("userRatedMovie%d" % k for k in range(2, T + 1))


def columns():
    from sparrowrecsys_b200 import features
    full = features.load_samples_csv(os.path.join(DATA, "trainingSamples.csv"))
    have = np.load(os.path.join(HERE, "deepfm_trainset.npz"))
    for k in ("movieId", "userId", "label"):
        assert np.array_equal(np.asarray(full[k], np.int64), have[k].astype(np.int64)), k
    rated1 = np.load(os.path.join(HERE, "widendeep_samples.npz"))["train_userRatedMovie1"]
    assert np.array_equal(np.asarray(full["userRatedMovie1"], np.int64), rated1.astype(np.int64))
    return {k: np.ascontiguousarray(full[k], np.int32) for k in HIST}


def load(part):
    """DIEN's feature dict of the train or test rows with their negatives (DIEN.py:49-50), from the committed
    fixtures."""
    from sparrowrecsys_b200.features import negative_history
    if part == "train":
        z = dict(np.load(os.path.join(HERE, "deepfm_trainset.npz")))
        z["userRatedMovie1"] = np.load(os.path.join(HERE, "widendeep_samples.npz"))["train_userRatedMovie1"]
        z.update(dict(np.load(os.path.join(HERE, "dien_train_samples.npz"))))
        seed = 2020
    else:
        z = dict(np.load(os.path.join(HERE, "dien_testset.npz")))
        seed = 2021
    z.update(negative_history(z, T, seed))
    return z


def evaluate(W, rows, batch):
    """`model.evaluate` of the oracle's weights over `rows` in batches of `batch`: {loss, auc, auc_value}."""
    from oracle import dien_train
    ps, zs, ys, auxs = [], [], [], []
    n = len(rows.mid)
    for lo in range(0, n, batch):
        r = rows.take(np.arange(lo, min(n, lo + batch)))
        p, z, aux, _ = dien_train.forward(W, r, np.float32)
        ps.append(p); zs.append(z); ys.append(r.y); auxs.append(aux)
    return dien_train.history_entry(ps, zs, ys, auxs)


def initial_weights(seed):
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_aux_weights, init_weights
    spec = default_spec("dien")
    return {**init_weights(spec, seed, for_test=False), **init_aux_weights(spec, seed)}


def run_seed(seed):
    from oracle import dien_train
    t0 = time.time()
    z = load("train")
    rows = dien_train.Rows.from_features(z, T)
    W, hist, opt = dien_train.fit(initial_weights(seed), rows, [np.arange(len(rows.mid))] * EPOCHS, BATCH,
                                  np.float32)
    seconds = time.time() - t0
    test = evaluate(W, dien_train.Rows.from_features(load("test"), T), BATCH)
    return {"seed": seed, "iterations": opt.iterations, "oracle_seconds": round(seconds, 1), "history": hist,
            "test": test}


def main():
    cols = columns()
    path = os.path.join(HERE, "dien_train_samples.npz")
    if "--check" in sys.argv:
        old = np.load(path)
        assert sorted(old.files) == sorted(cols), "columns differ from the committed file"
        assert all(old[k].dtype == cols[k].dtype and np.array_equal(old[k], cols[k]) for k in cols), \
            "columns differ from the committed file"
        print("dien train samples match")
        return
    np.savez_compressed(path, **cols)
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    with Pool(len(SEEDS)) as pool:
        runs = pool.map(run_seed, SEEDS)
    band = {k: [min(r["test"][k] for r in runs), max(r["test"][k] for r in runs)] for k in METRICS}
    res = {"rows": int(len(cols[HIST[0]])), "test_rows": int(len(load("test")["label"])), "epochs": EPOCHS,
           "batch_size": BATCH, "seeds": list(SEEDS), "runs": runs, "band": band}
    with open(os.path.join(HERE, "dien_fit.json"), "w") as f:
        json.dump(res, f, indent=1)
    for r in runs:
        print(r["seed"], r["oracle_seconds"], r["test"])
    print("band", band)


if __name__ == "__main__":
    main()
