"""Time the similar-movies catalogue build and query call on the GPU (`SimilarMovies`, csrc/similar.cu).

    python tools/similar_throughput.py [--repeats N] [--warmup W] [--out DIR]

Workloads (DESIGN.md section 4.23):
1. the reference's 982 movies and 203 150 ratings (tests/golden) with the shipped item2vec vectors: every movie as a
   query, size 10, with each ranker; the CPU oracle (oracle/similar_movies.py) is timed on the default ranker;
2. a seeded synthetic ML-20M-sized catalogue: 27 278 movies with 1 to 4 of 20 genres, 10^6 ratings, 16-dim vectors
   for 80 % of the movies; every movie as a query, size 10, with each ranker.
Times are the host clock around each synchronous call (upload, kernels and copies back), after --warmup calls: median,
min and max of --repeats.  The catalogue build is timed the same way.  The GPU's name and power limit are read in the
same run.  Prints one JSON document; --out also writes it to DIR/similar_throughput.json.
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


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "unavailable (%s)" % e
    return out


def timed(fn, warmup, repeats):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return {"median_ms": 1e3 * float(np.median(ts)), "min_ms": 1e3 * min(ts), "max_ms": 1e3 * max(ts)}


def reference_data():
    g = os.path.join(ROOT, "tests", "golden")
    from sparrowrecsys_b200.ranking import load_embeddings_csv
    m = np.load(os.path.join(g, "featureeng_movies.npz"))
    r = np.load(os.path.join(g, "featureeng_ratings.npz"))
    movies = {"movieId": m["movieId"].astype(np.int32), "genres": [str(x) for x in m["genres"]]}
    ratings = {"movieId": r["movieId"].astype(np.int32), "rating": r["half"].astype(np.float64) / 2}
    return movies, ratings, load_embeddings_csv(os.path.join(g, "item2vecEmb.csv"))


def synthetic_data(n=27_278, n_ratings=1_000_000, n_genres=20, dim=16, seed=0):
    rng = np.random.default_rng(seed)
    ids = np.arange(1, n + 1, dtype=np.int32)
    genres = ["|".join("G%d" % g for g in rng.choice(n_genres, rng.integers(1, 5), replace=False)) for _ in range(n)]
    ratings = {"movieId": ids[rng.integers(0, n, n_ratings)], "rating": rng.integers(1, 11, n_ratings) / 2}
    has = rng.random(n) < 0.8
    return {"movieId": ids, "genres": genres}, ratings, (ids[has], rng.standard_normal((int(has.sum()), dim))
                                                        .astype(np.float32))


def run(name, data, warmup, repeats, oracle=False):
    from sparrowrecsys_b200.similar import SimilarMovies
    movies, ratings, emb = data
    out = {"movies": len(movies["movieId"]), "ratings": int(len(ratings["movieId"])), "queries":
           len(movies["movieId"]), "size": 10}
    out["catalog_build"] = timed(lambda: SimilarMovies(movies, ratings, emb).close(), warmup, repeats)
    with SimilarMovies(movies, ratings, emb) as s:
        for model in ("default", "emb"):
            out["query_" + model] = timed(lambda: s.recommend_arrays(movies["movieId"], 10, model), warmup, repeats)
    if oracle:
        from oracle import similar_movies as S
        from sparrowrecsys_b200.similar import genre_lists
        t0 = time.perf_counter()
        c = S.Catalogue(movies["movieId"], genre_lists(movies["genres"]), ratings["movieId"],
                        np.asarray(ratings["rating"], np.float32))
        for mid in movies["movieId"].tolist():
            c.rec_list(mid, 10, "default")
        out["oracle_default_s"] = time.perf_counter() - t0
    print(name, json.dumps(out), file=sys.stderr)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"gpu": gpu_info(),
           "reference": run("reference", reference_data(), a.warmup, a.repeats, oracle=True),
           "synthetic_ml20m": run("synthetic", synthetic_data(), a.warmup, a.repeats)}
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "similar_throughput.json"), "w") as f:
            f.write(doc + "\n")


if __name__ == "__main__":
    main()
