"""Time NeuralCF's, the two towers', DeepFM's, Wide&Deep's, DeepFM_v2's or DIEN's `fit` on the GPU against the numpy
oracle on the host.

    python tools/fit_throughput.py [--model neuralcf|twotowers|deepfm|widendeep|deepfm_v2|dien] [--epochs 5]
                                   [--batch-sizes 12,4096]
                                   [--cpu-epochs 1] [--validate [--repeats 5]] [--kernels 4096]
                                   [--sample-weight [--repeats 5]]

Trains the reference script's run - the untrained model of `init_weights(default_spec(model), 0, for_test=False)`
over the 88 827 rows of `tests/golden/<model>_trainset.npz` (two towers: `neuralcf_trainset.npz`, and the model is
NeuralCF.py's neural_cf_model_2 with hidden_units [10, 10] and its final Dense; Wide&Deep: `deepfm_trainset.npz` with the columns of
`widendeep_samples.npz`; DeepFM_v2: `deepfm_trainset.npz`; DIEN: `deepfm_trainset.npz` with userRatedMovie1 of
`widendeep_samples.npz`, userRatedMovie2..5 of `dien_train_samples.npz`, the auxiliary head's initial weights and
the negatives of DIEN.py:49, in file order) - for `--epochs` epochs at each batch size, and reports
the wall time of `Trainer.fit` (upload, every step, the history read-back) and µs per step.  The CPU column is the
float32 oracle (`oracle.ncf_train.fit` / `oracle.twotowers_train.fit` / `oracle.deepfm_train.fit` / `oracle.widendeep_train.fit` /
`oracle.deepfm_v2_train.fit` / `oracle.dien_train.fit`) over `--cpu-epochs` epochs at the same batch
size, scaled to µs per step (`--cpu-epochs 0` leaves it out).  `--validate` adds the cost of validating on the
22 440 rows of `tests/golden/dien_testset.npz` every epoch, next to the epoch time: `validation_s_per_epoch` from
fits of `--val-epochs` one-step epochs (the first batch of rows) with and without validation, where the two validation
launches are a large part of each epoch, and `validated_minus_plain_s_per_epoch` from full-size fits (below the
noise of a 7 403-step epoch).  Plain and validated fits alternate, `--repeats` pairs, medians.  `--kernels B` adds
the device time of each kernel over one epoch at batch B (torch.profiler), per step.  `--sample-weight` adds the
step time of a fit with Keras sample weights (DESIGN.md section 4.28; seeded weights in [0, 2) with every tenth row
0) next to the unweighted one: `--repeats` alternating pairs of full fits, medians of µs per step.  Prints one JSON object with the card name and power limit read from nvidia-smi in the
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
    ap.add_argument("--model", choices=("neuralcf", "twotowers", "deepfm", "widendeep", "deepfm_v2", "dien"), default="neuralcf")
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--batch-sizes", default="12,4096")
    ap.add_argument("--cpu-epochs", type=int, default=1)
    ap.add_argument("--validate", action="store_true",
                    help="also report the cost per epoch of validating on dien_testset.npz every epoch")
    ap.add_argument("--val-epochs", type=int, default=500)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--kernels", type=int, default=0, help="batch size of a per-kernel breakdown (0: none)")
    ap.add_argument("--sample-weight", action="store_true",
                    help="also time fits with per-row sample weights, alternating with unweighted ones")
    args = ap.parse_args()
    dien = args.model == "dien"
    if dien and args.validate:
        ap.error("DIEN's fit takes no validation")
    if dien and args.sample_weight:
        ap.error("DIEN's fit takes no sample weights")
    from oracle import deepfm_train, deepfm_v2_train, dien_train, ncf_train, twotowers_train, widendeep_train
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.training import Trainer
    from sparrowrecsys_b200.weights import init_aux_weights, init_weights
    golden = os.path.join(ROOT, "tests", "golden")
    wd = args.model == "widendeep"
    ids_only = args.model in ("neuralcf", "twotowers")          # the models that read movieId and userId only
    z = np.load(os.path.join(golden, "%s_trainset.npz" % ("deepfm" if wd or args.model in ("deepfm_v2", "dien")
                                                          else "neuralcf" if ids_only else args.model)))
    if ids_only:
        feats = {k: z[k] for k in ("movieId", "userId", "label")}
    else:
        feats = dict(z)
    if wd:
        extra = np.load(os.path.join(golden, "widendeep_samples.npz"))
        feats.update({k[6:]: extra[k] for k in extra.files if k.startswith("train_")})
    if dien:
        from sparrowrecsys_b200.features import negative_history
        feats["userRatedMovie1"] = np.load(os.path.join(golden, "widendeep_samples.npz"))["train_userRatedMovie1"]
        feats.update(dict(np.load(os.path.join(golden, "dien_train_samples.npz"))))
        feats.update(negative_history(feats, 5, 2020))
    n = len(feats["label"])
    spec = default_spec(args.model, hidden=(10, 10), final_dense=True) if args.model == "twotowers" \
        else default_spec(args.model)
    W0 = init_weights(spec, 0, for_test=False)
    if dien:
        W0.update(init_aux_weights(spec, 0))

    def oracle_fit(orders, B):
        if ids_only:
            m = ncf_train if args.model == "neuralcf" else twotowers_train
            m.fit(W0, feats["movieId"], feats["userId"], feats["label"], orders, B, np.float32)
        elif dien:
            dien_train.fit(W0, dien_train.Rows.from_features(feats, 5), orders, B, np.float32)
        else:
            m = {"deepfm": deepfm_train, "widendeep": widendeep_train, "deepfm_v2": deepfm_v2_train}[args.model]
            m.fit(W0, m.Rows.from_features(feats), feats["label"], orders, B, np.float32)

    res = {"rows": n, "epochs": args.epochs, **card(), "runs": []}
    if args.model != "neuralcf":
        res = {"model": args.model, **res}
    val = None
    if args.validate:
        t = np.load(os.path.join(golden, "dien_testset.npz"))
        val = {k: t[k] for k in (("movieId", "userId", "label") if ids_only else t.files)}
        if wd:
            extra = np.load(os.path.join(golden, "widendeep_samples.npz"))
            val.update({k[5:]: extra[k] for k in extra.files if k.startswith("test_")})
        res["validation_rows"] = len(val["label"])

    weights = None
    if args.sample_weight:
        weights = np.random.default_rng(7).uniform(0.0, 2.0, n).astype(np.float32)
        weights[::10] = 0.0

    def timed_fit(B, validation_data=None, rows=None, epochs=args.epochs, sample_weight=None):
        f = feats if rows is None else {k: v[:rows] for k, v in feats.items()}
        with Trainer(spec, W0) as tr:
            t0 = time.perf_counter()
            hist = tr.fit(f, epochs=epochs, batch_size=B, seed=0, validation_data=validation_data,
                          sample_weight=sample_weight)
            return time.perf_counter() - t0, hist

    def paired(B, **kw):
        """median over --repeats alternating pairs of the validated fit's wall minus the plain fit's"""
        pairs = [(timed_fit(B, **kw)[0], timed_fit(B, val, **kw)[0]) for _ in range(args.repeats)]
        return float(np.median([p for p, _ in pairs])), float(np.median([v - p for p, v in pairs]))

    for B in (int(b) for b in args.batch_sizes.split(",")):
        steps = args.epochs * -(-n // B)
        with Trainer(spec, W0) as tr:
            tr.fit(feats, epochs=1, batch_size=B, seed=1, validation_data=val)   # warm-up: module load, first launches
        wall, hist = timed_fit(B)
        run = {"batch_size": B, "steps": steps, "gpu_wall_s": wall, "gpu_us_per_step": 1e6 * wall / steps}
        if val is not None:                       # plain and validated fits alternate, so drift hits both alike
            plain, extra = paired(B)
            _, extra_small = paired(B, rows=B, epochs=args.val_epochs)
            run.update({"gpu_epoch_s": plain / args.epochs, "validation_s_per_epoch": extra_small / args.val_epochs,
                        "validated_minus_plain_s_per_epoch": extra / args.epochs})
        if weights is not None:                   # unweighted and weighted fits alternate
            timed_fit(B, sample_weight=weights)   # warm-up of the weighted metrics kernel
            pairs = [(timed_fit(B)[0], timed_fit(B, sample_weight=weights)[0]) for _ in range(args.repeats)]
            plain = float(np.median([p for p, _ in pairs])) * 1e6 / steps
            weighted = float(np.median([w for _, w in pairs])) * 1e6 / steps
            run.update({"unweighted_us_per_step": plain, "weighted_us_per_step": weighted,
                        "weighted_over_unweighted": weighted / plain})
        if args.cpu_epochs:
            orders = [np.arange(n)] * args.cpu_epochs if dien else ncf_train.epoch_orders(n, args.cpu_epochs, 0)
            t0 = time.perf_counter()
            oracle_fit(orders, B)
            cpu = time.perf_counter() - t0
            cpu_steps = args.cpu_epochs * -(-n // B)
            run.update({"cpu_oracle_us_per_step": 1e6 * cpu / cpu_steps,
                        "cpu_oracle_wall_s_scaled": cpu * steps / cpu_steps})
        run["final_epoch"] = {k: v[-1] for k, v in hist.items()}
        res["runs"].append(run)
    if args.kernels:
        res["kernels"] = kernel_breakdown(spec, W0, feats, args.kernels)
    print(json.dumps(res))


def kernel_breakdown(spec, W0, feats, B):
    """{kernel: µs per step} of one epoch at batch B, from torch.profiler's CUDA activity (every kernel of the
    process, the library's included)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from sparrowrecsys_b200.training import Trainer
    n = len(feats["label"])
    steps = -(-n // B)
    with Trainer(spec, W0) as tr:
        tr.fit(feats, epochs=1, batch_size=B, seed=2)             # warm-up
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            tr.fit(feats, epochs=1, batch_size=B, seed=3)
    out = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in ev.name and "Memset" not in ev.name:
            name = ev.name.replace("(anonymous namespace)::", "").replace("void ", "").replace("srs::", "")
            name = name.split("(")[0].split("<")[0]
            out[name] = out.get(name, 0.0) + ev.device_time / steps
    return {"batch_size": B, "steps": steps, "us_per_step": dict(sorted(out.items(), key=lambda kv: -kv[1]))}


if __name__ == "__main__":
    main()
