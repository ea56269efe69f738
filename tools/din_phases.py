"""Where the DIN kernels spend their time at BASELINE cfg 3 (T = 50, E = 32, 4096-row batches).

    python tools/din_phases.py [--batches 64] [--launches 400]

Prints, for din_wg_kernel (din_impl=tc) and din_kernel (din_impl=cudacore):
  * the share of cycles per phase (srs::DinPhase, csrc/common.cuh) on bench's inputs, from a phase-timing
    build of the library (-DSRS_DIN_PHASES) compiled into a temporary directory - the in-tree library is
    untouched;
  * the kernel time per batch with CUDA events over many launches of the in-tree library, in bench.py's
    default mode (two streams, each launch capped to SMs / 2 CTAs) and on a single stream, for four sets
    of history ids with the same shapes and the same number of row gathers (INPUTS): bench's Zipf ids
    with 0-padded histories, Zipf ids with every history full, and uniform ids padded and full.  Zipf
    ids and padding make a few table rows hot (half of bench's history positions read row 0); uniform
    full histories spread the reads over the whole table, so the sets show what reuse of rows costs;
  * the card name and power limit.
Needs a GPU.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["tile inputs", "W_r / folded column", "gather issue", "gather wait", "AU MMA", "gate", "pooling",
          "AU position loop", "row imbalance", "top MLP", "image wait"]
IMPLS = (("tc", "din_wg_kernel"), ("cudacore", "din_kernel"))
# name -> synthetic_features options; the first is bench's inputs
INPUTS = (("zipf, padded", {}),
          ("zipf, full", {"pad_history": False}),
          ("uniform, padded", {"uniform_history": True}),
          ("uniform, full", {"uniform_history": True, "pad_history": False}))


def make_ring(n_batches, B, seed=1, **history):
    """n_batches distinct cfg 3 batches in HBM (together larger than the L2), and a cfg 3 model per impl.
    `history`: synthetic_features' options for the history ids (INPUTS)."""
    import torch
    from sparrowrecsys_b200.features import synthetic_features
    from sparrowrecsys_b200.spec import baseline_spec
    from sparrowrecsys_b200.weights import init_weights
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 2)
    feats = synthetic_features(spec, n_batches * B, seed=seed, **history)
    batches = [{k: v[i * B:(i + 1) * B] for k, v in feats.items()} for i in range(n_batches)]
    return spec, W, batches, torch


def phases(args):
    """Child process: runs against the phase-timing build named by SRS_CTR_LIB."""
    from sparrowrecsys_b200.model import CTRModel
    spec, W, batches, torch = make_ring(args.batches, args.batch)
    out = {}
    for impl, name in IMPLS:
        with CTRModel(spec, W, device=0, options={"din_impl": impl}) as m:
            assert m.kernel_name == name, m.kernel_name
            dev = [m.to_device(b) for b in batches]
            probs = torch.empty(args.batch, dtype=torch.float32, device="cuda:0")
            fn = m._lib.srs_debug_din_phases
            fn.restype = C.c_int
            fn.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int32]
            cyc = (C.c_uint64 * 16)()
            for i in range(len(dev)):                       # warm-up, then clear the counters
                m.predict_device(dev[i], probs)
            fn(m._h, cyc, 16)
            for i in range(args.launches):
                m.predict_device(dev[i % len(dev)], probs)
            m.status()
            fn(m._h, cyc, 16)
            tot = sum(cyc[i] for i in range(len(PHASES)))
            out[name] = {PHASES[i]: round(100.0 * cyc[i] / max(tot, 1), 1) for i in range(len(PHASES)) if cyc[i]}
    print(json.dumps(out))


def timing(args, history):
    """Kernel time per batch of the in-tree library: CUDA events around `launches` launches."""
    from sparrowrecsys_b200.model import CTRModel
    spec, W, batches, torch = make_ring(args.batches, args.batch, **history)
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = {}
    for impl, name in IMPLS:
        with CTRModel(spec, W, device=0, options={"din_impl": impl}) as m:
            dev = [m.to_device(b) for b in batches]
            probs = [torch.empty(args.batch, dtype=torch.float32, device="cuda:0") for _ in range(2)]
            streams = [torch.cuda.Stream() for _ in range(2)]
            for mode, n_streams, limit in (("2 streams, SMs/2 CTAs per launch", 2, n_sms // 2),
                                           ("1 stream, no SM limit", 1, 0)):
                m.set_sm_limit(limit)
                main = torch.cuda.current_stream()

                def run(n):
                    for s in streams[:n_streams]:
                        s.wait_stream(main)
                    for i in range(n):
                        k = i % n_streams
                        m.predict_device(dev[i % len(dev)], probs[k], stream=streams[k])
                    for s in streams[:n_streams]:
                        main.wait_stream(s)

                run(2 * len(dev))
                torch.cuda.synchronize()
                times = []
                for _ in range(5):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(main)
                    run(args.launches)
                    e1.record(main)
                    e1.synchronize()
                    times.append(1e3 * e0.elapsed_time(e1) / args.launches)
                m.status()
                times.sort()
                res.setdefault(name, {})[mode] = {"us_per_batch_median": round(times[2], 2),
                                                  "min": round(times[0], 2), "max": round(times[-1], 2),
                                                  "M_inf_per_s": round(args.batch / times[2], 1)}
            m.set_sm_limit(0)
    return res


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = "nvidia-smi failed: %r" % (e,)
    return q


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--batches", type=int, default=64, help="distinct batches resident in HBM")
    ap.add_argument("--launches", type=int, default=400)
    ap.add_argument("--phases-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.phases_child:
        return phases(args)
    from sparrowrecsys_b200 import build
    build.build()
    print(json.dumps({"card": card()}))
    for name, history in INPUTS:
        print(json.dumps({"kernel_time": timing(args, history), "history": name}))
    with tempfile.TemporaryDirectory(prefix="srs_din_phases_") as tmp:
        lib = build.build(defines=["SRS_DIN_PHASES"], out_dir=tmp)
        env = dict(os.environ, SRS_CTR_LIB=lib)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--phases-child",
                            "--batch", str(args.batch), "--batches", str(args.batches),
                            "--launches", str(min(args.launches, 100))],
                           env=env, capture_output=True, text=True)
        sys.stderr.write(r.stderr)
        if r.returncode != 0:
            raise SystemExit("phase-timing run failed (exit %d)" % r.returncode)
        print(json.dumps({"phase_share_percent": json.loads(r.stdout.strip().splitlines()[-1])}))


if __name__ == "__main__":
    main()
