"""Time NeuralCF's or DeepFM's `fit` on the GPU against the numpy oracle on the host.

    python tools/fit_throughput.py [--model neuralcf|deepfm] [--epochs 5] [--batch-sizes 12,4096] [--cpu-epochs 1]

Trains the reference script's run - the untrained model of `init_weights(default_spec(model), 0, for_test=False)`
over the 88 827 rows of `tests/golden/<model>_trainset.npz` - for `--epochs` epochs at each batch size, and reports
the wall time of `Trainer.fit` (upload, every step, the history read-back) and µs per step.  The CPU column is the
float32 oracle (`oracle.ncf_train.fit` / `oracle.deepfm_train.fit`) over `--cpu-epochs` epochs at the same batch
size, scaled to µs per step.  Prints one JSON object with the card name and power limit read from nvidia-smi in the
same run (and the model's name unless it is the default, NeuralCF).  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:                         # the numbers stand without it, marked as such
        return {"gpu": "not reported (%s)" % type(e).__name__, "power_limit": "not reported"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=("neuralcf", "deepfm"), default="neuralcf")
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--batch-sizes", default="12,4096")
    ap.add_argument("--cpu-epochs", type=int, default=1)
    args = ap.parse_args()
    from oracle import deepfm_train, ncf_train
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.training import Trainer
    from sparrowrecsys_b200.weights import init_weights
    z = np.load(os.path.join(ROOT, "tests", "golden", "%s_trainset.npz" % args.model))
    if args.model == "neuralcf":
        feats = {k: z[k] for k in ("movieId", "userId", "label")}
    else:
        feats = dict(z)
    n = len(feats["label"])
    spec = default_spec(args.model)
    W0 = init_weights(spec, 0, for_test=False)

    def oracle_fit(orders, B):
        if args.model == "neuralcf":
            ncf_train.fit(W0, feats["movieId"], feats["userId"], feats["label"], orders, B, np.float32)
        else:
            deepfm_train.fit(W0, deepfm_train.Rows.from_features(feats), feats["label"], orders, B, np.float32)

    res = {"rows": n, "epochs": args.epochs, **card(), "runs": []}
    if args.model != "neuralcf":
        res = {"model": args.model, **res}
    for B in (int(b) for b in args.batch_sizes.split(",")):
        steps = args.epochs * -(-n // B)
        with Trainer(spec, W0) as tr:
            tr.fit(feats, epochs=1, batch_size=B, seed=1)          # warm-up: module load, first launches
        with Trainer(spec, W0) as tr:
            t0 = time.perf_counter()
            hist = tr.fit(feats, epochs=args.epochs, batch_size=B, seed=0)
            wall = time.perf_counter() - t0
        orders = ncf_train.epoch_orders(n, args.cpu_epochs, 0)
        t0 = time.perf_counter()
        oracle_fit(orders, B)
        cpu = time.perf_counter() - t0
        cpu_steps = args.cpu_epochs * -(-n // B)
        res["runs"].append({"batch_size": B, "steps": steps, "gpu_wall_s": wall, "gpu_us_per_step": 1e6 * wall / steps,
                            "cpu_oracle_us_per_step": 1e6 * cpu / cpu_steps,
                            "cpu_oracle_wall_s_scaled": cpu * steps / cpu_steps,
                            "final_epoch": {k: v[-1] for k, v in hist.items()}})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
