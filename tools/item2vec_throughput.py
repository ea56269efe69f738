"""Time item2vec training on the GPU (`embedding.item2vec`) against the C oracle's single-threaded run.

    python tools/item2vec_throughput.py [--partitions 1,33,132,528,1056] [--skip-corpus] [--skip-synthetic] [--out DIR]

Two workloads: the corpus fixture (tests/golden/item2vec_corpus.npz: the reference's 657 069 positive ratings) at the
script's configuration (vector size 10, window 5, 10 iterations), and a seeded synthetic ML-20M-sized set (20 M
ratings, 27 278 movies, 138 493 users, Zipf-like movie popularity and user activity) at 2 iterations.  For each
partition count P: the wall time of a whole call (host clock around a synchronous call), the time per iteration
(the difference between a run of I iterations and one of 1, over I - 1: sentence building and the copies cancel),
the words trained per second, and the mean top-10 cosine-neighbour overlap with the P = 1 result over the 1 000 most
frequent movies (Spark's averaging of the partitions' tables costs quality as P grows).  The C oracle's P = 1 time is
taken once per workload on this host's CPU.  The GPU's name and power limit are read in the same call.  Prints one
JSON document; --out also writes it to DIR/item2vec_throughput.json.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "unavailable (%s)" % e
    return out


def synthetic_ml20m(seed=20):
    """20 M ratings: user activity and movie popularity both Zipf-like, half-stars with MovieLens-like weights,
    timestamps of 9 and 10 digits."""
    rng = np.random.default_rng(seed)
    n, n_users, n_movies = 20000000, 138493, 27278
    w_user = 1.0 / (np.arange(n_users) + 20.0)
    per_user = rng.multinomial(n - 20 * n_users, w_user / w_user.sum()) + 20
    user = np.repeat(np.arange(1, n_users + 1, dtype=np.int32), per_user)
    w_movie = 1.0 / (np.arange(n_movies) + 5.0) ** 1.1
    movie = (rng.choice(n_movies, n, p=w_movie / w_movie.sum()) + 1).astype(np.int32)
    half = rng.choice(np.arange(1, 11), n, p=np.array([1, 3, 2, 7, 5, 21, 12, 27, 8, 14]) / 100.0)
    ts = rng.integers(789652009, 1427784002, n).astype(np.int32)
    return {"userId": user, "movieId": movie, "rating": half / 2.0, "timestamp": ts}


def top10(vec, queries):
    x = vec.astype(np.float64)
    x /= np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-30)
    s = x[:queries] @ x.T
    s[np.arange(queries), np.arange(queries)] = -np.inf
    return np.argsort(-s, axis=1, kind="stable")[:, :10]


def overlap(a, b):
    return float(np.mean([len(set(x) & set(y)) / 10.0 for x, y in zip(a.tolist(), b.tolist())]))


def workload(name, ratings, iterations, partitions, repeats):
    from oracle import item2vec as I
    from oracle import item2vec_cext as X
    from sparrowrecsys_b200 import embedding as E
    half = np.rint(np.asarray(ratings["rating"]) * 2).astype(np.int64)
    _, seqs = I.positive_sequences(ratings["userId"], ratings["movieId"], half, ratings["timestamp"])
    ids, counts = I.build_vocab(seqs)
    words, offs = I.chunk_corpus(seqs, ids)
    code, point, codelen = I.huffman(counts)
    t0 = time.perf_counter()
    X.train(words, offs, counts, code, point, codelen, 10, 5, 1, 1, 0)
    oracle_iter = time.perf_counter() - t0
    res = {"workload": name, "ratings": int(len(half)), "words": int(len(words)), "vocabulary": int(len(ids)),
           "deepest_code": int(codelen.max()), "iterations": iterations,
           "c_oracle_seconds_per_iteration_P1": round(oracle_iter, 3), "runs": []}
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}), flush=True)
    E.item2vec({k: v[:20000] for k, v in ratings.items()}, num_iterations=1)   # warm-up: module load, allocator
    q = min(1000, len(ids))
    base = None
    for P in partitions:
        t_full, t_one = [], []
        for _ in range(repeats):
            t0 = time.perf_counter()
            ids_p, vec = E.item2vec(ratings, num_iterations=iterations, num_partitions=P)
            t_full.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            E.item2vec(ratings, num_iterations=1, num_partitions=P)
            t_one.append(time.perf_counter() - t0)
        full, one = float(np.median(t_full)), float(np.median(t_one))
        per_iter = (full - one) / (iterations - 1)
        nb = top10(vec, q)
        if base is None:
            base = nb
        res["runs"].append({"partitions": P, "call_seconds": round(full, 3), "call_seconds_1_iteration": round(one, 3),
                            "seconds_per_iteration": round(per_iter, 4),
                            "words_per_second": round(len(words) / per_iter if per_iter > 0 else float("nan")),
                            "speedup_vs_c_oracle_P1": round(oracle_iter / per_iter, 2) if per_iter > 0 else None,
                            "top10_overlap_with_P1": round(overlap(nb, base), 4)})
        print(json.dumps(res["runs"][-1]), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--partitions", default="1,33,132,528,1056")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--skip-synthetic", action="store_true")
    ap.add_argument("--skip-corpus", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool measures the GPU and has no CPU fallback")
    from test_item2vec_oracle import corpus_ratings
    parts = [int(x) for x in a.partitions.split(",")]
    doc = {"gpu": gpu_info(), "workloads": []}
    print(json.dumps({"gpu": doc["gpu"]}), flush=True)
    if not a.skip_corpus:
        doc["workloads"].append(workload("corpus fixture", corpus_ratings(), 10, parts, a.repeats))
    if not a.skip_synthetic:
        doc["workloads"].append(workload("synthetic ML-20M", synthetic_ml20m(), 2, parts, 1))
    doc["gpu_after"] = gpu_info()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "item2vec_throughput.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
