"""Time DeepWalk's walks, its Word2Vec stage and the bucketed random-projection LSH on the GPU (`embedding`) against
the numpy / C oracles on the host.

    python tools/graph_lsh_throughput.py [--skip-synthetic] [--skip-lsh-synthetic] [--out DIR]

Workloads (DESIGN.md section 4.14):
* the reference's corpus (tests/golden/item2vec_corpus.npz): transitions + 20 000 walks of length 10
  (`random_walks`) against oracle/graphemb.py; the Word2Vec stage (10 iterations, P = 1) as a whole
  `graph_embedding` call minus the `random_walks` call, against oracle/item2vec_c.c on the oracle's walks;
* the seeded synthetic ML-20M-sized set of tools/featureeng_throughput.py: transitions + 10^6 walks of length 10;
* LSH over 10^6 seeded N(0, 1) 64-dim float32 vectors, 3 tables, bucket length 0.1: `transform`, and
  `approx_nearest_neighbors` of 10^4 keys (k = 5) in one call; the oracle's query time is taken on a few keys and
  scaled (reported as such);
* LSH over the 881 shipped item2vec vectors with every movie as a key (k = 5), the reference's settings.
Times are the host clock around synchronous calls, the median of --repeats; the GPU's name and power limit are read
in the same call.  Prints one JSON document; --out also writes it to DIR/graph_lsh_throughput.json.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "unavailable (%s)" % e
    return out


def timed(f, repeats):
    ts = []
    out = None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = f()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def walks_workload(name, r, num_walks, repeats, word2vec):
    from oracle import graphemb as G
    from oracle import item2vec as I
    from oracle import item2vec_cext as X
    from sparrowrecsys_b200 import embedding as E
    from test_item2vec_oracle import halves
    t_gpu, (w, n) = timed(lambda: E.random_walks(r, num_walks, 10), repeats)
    t0 = time.perf_counter()
    _, seqs = I.positive_sequences(r["userId"], r["movieId"], halves(r), r["timestamp"])
    t_seq = time.perf_counter() - t0
    t0 = time.perf_counter()
    tr = G.transitions(seqs)
    ow, on = G.random_walks(tr, num_walks, 10)
    t_or = time.perf_counter() - t0
    res = {"workload": name, "ratings": int(len(r["userId"])), "sources": int(len(tr["sources"])),
           "distinct_pairs": int(len(tr["targets"])), "walks": num_walks, "walk_length": 10,
           "gpu_transitions_and_walks_seconds": round(t_gpu, 4),
           "oracle_sentences_seconds": round(t_seq, 3), "oracle_transitions_and_walks_seconds": round(t_or, 3),
           "walks_equal_oracle": bool(np.array_equal(w, ow) and np.array_equal(n, on)),
           "walks_speedup_vs_oracle_excluding_its_sentences": round(t_or / t_gpu, 1)}
    print(json.dumps(res), flush=True)
    if word2vec:
        t_all, (ids, vec) = timed(lambda: E.graph_embedding(r, num_walks=num_walks), 1)
        sents = G.walk_sentences(ow, on)
        vids, counts = I.build_vocab(sents)
        words, offs = I.chunk_corpus(sents, vids)
        code, point, codelen = I.huffman(counts)
        t0 = time.perf_counter()
        ovec = X.train(words, offs, counts, code, point, codelen, 10, 5, 10, 1, 0)
        t_c = time.perf_counter() - t0
        res.update({"walk_words": int(len(words)), "gpu_graph_embedding_call_seconds": round(t_all, 3),
                    "gpu_word2vec_stage_seconds": round(t_all - t_gpu, 3),
                    "c_oracle_word2vec_seconds": round(t_c, 3),
                    "graph_embedding_equals_c_oracle": bool(np.array_equal(vec.view(np.int32),
                                                                           ovec.view(np.int32)))})
        print(json.dumps(res), flush=True)
    return res


def lsh_workload(name, ids, x, keys, bl, tables, k, repeats, oracle_keys):
    from oracle import lsh as H
    from sparrowrecsys_b200 import embedding as E
    model = E.BucketedRandomProjectionLSH(bucket_length=bl, num_hash_tables=tables).fit(x)
    t_tr, b = timed(lambda: model.transform(x), repeats)
    t_q, res_q = timed(lambda: model.approx_nearest_neighbors(ids, x, keys, k), repeats)
    uv = model.rand_unit_vectors
    t0 = time.perf_counter()
    ob = H.transform(x, uv, bl)
    t_otr = time.perf_counter() - t0
    nk = min(oracle_keys, len(keys))
    t0 = time.perf_counter()
    same = True
    for q in range(nk):
        oi, od = H.approx_nearest_neighbors(ids, x, uv, bl, keys[q], k)
        same &= bool(np.array_equal(oi, res_q[q][0]) and np.array_equal(od, res_q[q][1]))
    t_oq = (time.perf_counter() - t0) * len(keys) / nk
    res = {"workload": name, "rows": int(len(x)), "dim": int(x.shape[1]), "tables": tables, "bucket_length": bl,
           "keys": int(len(keys)), "k": k, "gpu_transform_seconds": round(t_tr, 4),
           "gpu_query_seconds": round(t_q, 4), "oracle_transform_seconds": round(t_otr, 3),
           "oracle_query_seconds": round(t_oq, 3), "oracle_query_keys_timed": nk,
           "mean_candidates_first_keys": None,
           "buckets_equal_oracle": bool(np.array_equal(b, ob)), "queries_equal_oracle_on_timed_keys": same,
           "transform_speedup_vs_oracle": round(t_otr / t_tr, 1), "query_speedup_vs_oracle": round(t_oq / t_q, 1)}
    kb = H.transform(keys[:nk], uv, bl)
    res["mean_candidates_first_keys"] = float(np.mean([np.sum(np.any(ob == kb[q], axis=1)) for q in range(nk)]))
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--skip-synthetic", action="store_true")
    ap.add_argument("--skip-lsh-synthetic", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool measures the GPU and has no CPU fallback")
    from sparrowrecsys_b200 import embedding as E
    from test_item2vec_oracle import corpus_ratings, shipped_items
    doc = {"gpu": gpu_info(), "workloads": []}
    print(json.dumps({"gpu": doc["gpu"]}), flush=True)
    ref = corpus_ratings()
    E.random_walks({k: v[:5000] for k, v in ref.items()}, 10, 10)     # warm-up: module load, context
    doc["workloads"].append(walks_workload("reference corpus", ref, 20000, a.repeats, True))
    sid, svec = shipped_items()
    doc["workloads"].append(lsh_workload("shipped item2vec vectors, every movie a key", sid, svec,
                                         svec.astype(np.float64), 0.1, 3, 5, a.repeats, len(sid)))
    if not a.skip_lsh_synthetic:
        rng = np.random.default_rng(0)
        x = rng.standard_normal((1000000, 64)).astype(np.float32)
        keys = rng.standard_normal((10000, 64))
        doc["workloads"].append(lsh_workload("synthetic 10^6 x 64", np.arange(len(x), dtype=np.int32), x, keys,
                                             0.1, 3, 5, 1, 3))
    if not a.skip_synthetic:
        from featureeng_throughput import synthetic_ml20m
        doc["workloads"].append(walks_workload("synthetic ML-20M", synthetic_ml20m()[0], 1000000, 1, False))
    doc["gpu_after"] = gpu_info()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "graph_lsh_throughput.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
