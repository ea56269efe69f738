"""Cost of DIEN's auxiliary head on the H100.

    python tools/dien_aux_cost.py [--iters 200] [--rounds 5]

For E = 10 / T = 5 (the reference script's shape) and E = 32 / T = 50, B = 4096: a CUDA graph of `iters`
launches of the plain forward (`srs_predict_device`, dien_kernel<EP, false>) against one of the two-output
call (`srs_dien_outputs_device`: dien_kernel<EP, true> and the final-loss kernel) on the same device batch.
The graphs alternate, `rounds` times each, timed with CUDA events; the medians are reported per batch.  The
two calls' probabilities are checked to be bit-identical first.  Prints one JSON object with the card name
and power limit read from nvidia-smi.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

from eval_throughput import card          # noqa: E402


def measure(E, T, B, iters, rounds):
    import torch
    from sparrowrecsys_b200 import _lib
    from sparrowrecsys_b200.features import negative_history, negative_history_keys, synthetic_features
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_aux_weights, init_weights
    spec = default_spec("dien", emb_dim=E, hist_len=T)
    m = CTRModel(spec, {**init_weights(spec, 1), **init_aux_weights(spec, 1)})
    feats = synthetic_features(spec, B, seed=1)
    negs = negative_history(feats, T, seed=1, n_movies=spec.n_movies)
    db = m.to_device(feats)
    neg = torch.from_numpy(np.ascontiguousarray(
        np.stack([negs[k] for k in negative_history_keys(T)], axis=1))).cuda()
    lab = torch.from_numpy((np.arange(B) % 2).astype(np.int32)).cuda()
    probs, logits, aux, final, probs2 = (torch.empty(B, device="cuda") for _ in range(5))
    s = torch.cuda.Stream()
    b = db.struct()

    def plain():
        m.predict_device(db, probs, logits, stream=s)

    def two_outputs():
        _lib.check(m._lib.srs_dien_outputs_device(m._h, C.byref(b), neg.data_ptr(), T - 1, lab.data_ptr(),
                                                  probs2.data_ptr(), logits.data_ptr(), aux.data_ptr(),
                                                  final.data_ptr(), s.cuda_stream))
    with torch.cuda.stream(s):
        plain()
        two_outputs()
    s.synchronize()
    m.status()
    assert torch.equal(probs, probs2), "the AUX variant changed y_pred"
    graphs = {}
    for name, f in (("plain", plain), ("aux", two_outputs)):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(iters):
                f()
        graphs[name] = g
    times = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():                # alternate
            g.replay()
            torch.cuda.synchronize()
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g.replay()
            e.record()
            e.synchronize()
            times[k].append(a.elapsed_time(e) * 1e3 / iters)
    med = {k: float(np.median(v)) for k, v in times.items()}
    m.close()
    return {"E": E, "T": T, "B": B, "us_per_batch_plain": med["plain"], "us_per_batch_aux": med["aux"],
            "added_fraction": (med["aux"] - med["plain"]) / med["plain"], "runs_us": times}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    out = dict(card())
    out["shapes"] = [measure(10, 5, 4096, a.iters, a.rounds), measure(32, 50, 4096, a.iters, a.rounds)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
