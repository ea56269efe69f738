"""Time multi-channel and embedding recall on the GPU (`SimilarMovies.recommend(..., candidates="multiple")` and
`SimilarMovies.retrieve_by_embedding`, csrc/similar.cu).

    python tools/recall_throughput.py [--repeats N] [--warmup W] [--out DIR]

Workloads (DESIGN.md section 4.24), every movie of the catalogue a query:
1. the reference's 982 movies and 203 150 ratings (tests/golden) with their titles and the shipped item2vec vectors;
2. a seeded synthetic ML-20M-sized catalogue (tests/test_gpu_similar_recall.py's): 27 278 movies with ids up to
   131 262 in a shuffled load order, so HashMap order is not id order, heavy ties in years and ratings, 16-dim vectors
   for 80 % of the movies.
Each is timed with multi-channel recall under both rankers at size 10, and embedding recall at sizes 10 and 2 000.
Times are the host clock around each synchronous call (upload, kernels and copies back), after --warmup calls:
median, min and max of --repeats.  The catalogue build is timed the same way.  The GPU's name and power limit are
read in the same run.  Prints one JSON document; --out also writes it to DIR/recall_throughput.json.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from similar_throughput import gpu_info, timed  # noqa: E402


def reference_data():
    from sparrowrecsys_b200.ranking import load_embeddings_csv
    g = os.path.join(ROOT, "tests", "golden")
    m = np.load(os.path.join(g, "featureeng_movies.npz"))
    r = np.load(os.path.join(g, "featureeng_ratings.npz"))
    movies = {"movieId": m["movieId"].astype(np.int32), "genres": [str(x) for x in m["genres"]],
              "title": [str(x) for x in m["title"]]}
    ratings = {"movieId": r["movieId"].astype(np.int32), "rating": r["half"].astype(np.float64) / 2}
    return movies, ratings, load_embeddings_csv(os.path.join(g, "item2vecEmb.csv"))


def synthetic_data():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_similar_recall import synthetic_catalogue
    return synthetic_catalogue()


def run(name, data, warmup, repeats):
    from sparrowrecsys_b200.similar import SimilarMovies
    movies, ratings, emb = data
    q = movies["movieId"]
    out = {"movies": len(q), "ratings": int(len(ratings["movieId"])), "vectors": int(len(emb[0])), "queries": len(q)}
    out["catalog_build"] = timed(lambda: SimilarMovies(movies, ratings, emb).close(), warmup, repeats)
    with SimilarMovies(movies, ratings, emb) as s:
        for model in ("default", "emb"):
            out["multiple_%s_size10" % model] = timed(lambda: s.recommend_arrays(q, 10, model, "multiple"), warmup,
                                                      repeats)
        for size in (10, 2000):
            out["embedding_recall_size%d" % size] = timed(lambda: s.retrieve_by_embedding_arrays(q, size), warmup,
                                                          repeats)
    print(name, json.dumps(out), file=sys.stderr)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"gpu": gpu_info(),
           "reference": run("reference", reference_data(), a.warmup, a.repeats),
           "synthetic_ml20m": run("synthetic", synthetic_data(), a.warmup, a.repeats)}
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "recall_throughput.json"), "w") as f:
            f.write(doc + "\n")


if __name__ == "__main__":
    main()
