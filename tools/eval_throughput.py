"""Cost of `evaluate`'s metrics on the H100.

    python tools/eval_throughput.py [--iters 200] [--rounds 3]

* Device path: a CUDA graph of `predict_device` alone against one of `predict_device` +
  `Metrics.update_device` on the same batch, for BASELINE cfg 3 DIN (B = 4096, T = 50) and NeuralCF
  (B = 4096); the difference is the metrics kernel's added time per batch.
* Host path: `evaluate` rows/s against `predict_host_batches` (`predict(batch_size=...)`) on the same
  batches.

Runs alternate between the variants, each timed with CUDA events (host path: wall clock around the
synchronous call).  Prints one JSON object with the card name and power limit read from nvidia-smi.
Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:                         # the numbers stand without it, marked as such
        return {"gpu": "not reported (%s)" % type(e).__name__, "power_limit": "not reported"}


def device_path(name, spec, iters, rounds):
    import torch
    from sparrowrecsys_b200.features import synthetic_features
    from sparrowrecsys_b200.model import CTRModel, Metrics
    from sparrowrecsys_b200.weights import init_weights
    B = 4096
    m = CTRModel(spec, init_weights(spec, 1))
    mt = Metrics(0)
    feats = synthetic_features(spec, B, seed=1)
    db = m.to_device(feats)
    probs = torch.empty(B, device="cuda")
    logits = torch.empty(B, device="cuda")
    lab = torch.from_numpy((np.arange(B) % 2).astype(np.int32)).cuda()
    s = torch.cuda.Stream()
    graphs = {}
    for variant in ("predict", "predict+metrics"):
        with torch.cuda.stream(s):                 # warm-up outside capture
            m.predict_device(db, probs, logits, stream=s)
            if variant != "predict":
                mt.update_device(probs, logits, lab, stream=s)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(iters):
                m.predict_device(db, probs, logits, stream=s)
                if variant != "predict":
                    mt.update_device(probs, logits, lab, stream=s)
        graphs[variant] = g
    times = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():                # alternate
            g.replay()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g.replay()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) * 1e3 / iters)
    med = {k: float(np.median(v)) for k, v in times.items()}
    mt.close()
    m.close()
    return {"model": name, "B": B, "us_per_batch_predict": med["predict"],
            "us_per_batch_predict_metrics": med["predict+metrics"],
            "metrics_added_us": med["predict+metrics"] - med["predict"],
            "added_fraction": (med["predict+metrics"] - med["predict"]) / med["predict"],
            "runs_us": times}


def host_path(name, spec, n, batch, rounds):
    from sparrowrecsys_b200.features import synthetic_features
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.weights import init_weights
    m = CTRModel(spec, init_weights(spec, 1))
    feats = synthetic_features(spec, n, seed=2)
    feats["label"] = (np.arange(n) % 2).astype(np.int32)
    calls = {"predict_host_batches": lambda: m.predict(feats, batch_size=batch),
             "evaluate": lambda: m.evaluate(feats, batch_size=batch)}
    for f in calls.values():
        f()
    times = {k: [] for k in calls}
    for _ in range(rounds):
        for k, f in calls.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)
    m.close()
    return {"model": name, "rows": n, "batch": batch,
            **{"rows_per_s_" + k: n / float(np.median(v)) for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    from sparrowrecsys_b200.spec import baseline_spec, default_spec
    din, ncf = baseline_spec("cfg3_din"), default_spec("neuralcf")
    out = dict(card())
    out["device_path"] = [device_path("din_cfg3", din, a.iters, a.rounds),
                          device_path("neuralcf", ncf, a.iters, a.rounds)]
    out["host_path"] = [host_path("din_cfg3", din, 200_000, 4096, a.rounds),
                        host_path("neuralcf", ncf, 1_000_000, 4096, a.rounds)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
