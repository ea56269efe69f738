"""Users per second of the "Recommended for you" page on the GPU (`RecForYou`, csrc/recforyou.cu), with each ranker.

    python tools/recforyou_throughput.py [--repeats N] [--warmup W] [--oracle-users N] [--out DIR]

Workloads (DESIGN.md section 4.25), every user of the ratings answered in one call at size 20:
1. reference: the 982 movies, 203 150 ratings and 5 000 users of tests/golden, the shipped item2vec and userEmb
   vectors and, for "nerualcf", the shipped NeuralCF model (neuralcf_002);
2. synthetic: a seeded catalogue of 27 278 movies with 10^6 ratings by 30 000 users, 16-dim vectors for 80 % of the
   movies and 70 % of the users, and a NeuralCF model of the reference's shape over those ids.
GPU times are the host clock around each synchronous call (upload, kernels and copies back), after --warmup calls:
median, min and max of --repeats; users/s is users over the median.  The CPU column is the oracle
(oracle/recforyou.py) timed on the first --oracle-users users of the same call.  The GPU's name and power limit are
read in the same run.  Prints one JSON line per workload and ranker; --out also writes them to
DIR/recforyou_throughput.jsonl.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from similar_throughput import gpu_info, timed  # noqa: E402

SIZE = 20
RANKERS = ("default", "emb", "nerualcf")


def reference_data():
    g = os.path.join(ROOT, "tests", "golden")
    from sparrowrecsys_b200.ranking import load_embeddings_csv
    from sparrowrecsys_b200.spec import default_spec
    m = np.load(os.path.join(g, "featureeng_movies.npz"))
    r = np.load(os.path.join(g, "featureeng_ratings.npz"))
    movies = {"movieId": m["movieId"].astype(np.int32), "genres": [str(x) for x in m["genres"]]}
    ratings = {"userId": r["userId"].astype(np.int32), "movieId": r["movieId"].astype(np.int32),
               "rating": r["half"].astype(np.float64) / 2}
    z = np.load(os.path.join(g, "item2vec_user_emb.npz"))
    uemb = (z["user"].astype(np.int32),
            np.array([[float(v) for v in ln.split(":")[1].split()] for ln in z["line"].tolist()], np.float32))
    w = np.load(os.path.join(g, "neuralcf_002.npz"))
    W = {k.replace("__", "/"): w[k] for k in w.files if k not in ("user_ids", "user_rows")}
    W["userId_embedding"] = np.zeros((30001, w["user_rows"].shape[1]), np.float32)
    W["userId_embedding"][w["user_ids"]] = w["user_rows"]
    return movies, ratings, load_embeddings_csv(os.path.join(g, "item2vecEmb.csv")), uemb, default_spec("neuralcf"), W


def synthetic_data(n=27_278, n_users=30_000, n_ratings=1_000_000, dim=16, seed=0):
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    rng = np.random.default_rng(seed)
    ids = np.arange(1, n + 1, dtype=np.int32)
    genres = ["|".join("G%d" % g for g in rng.choice(20, rng.integers(1, 5), replace=False)) for _ in range(n)]
    users = np.arange(1, n_users + 1, dtype=np.int32)
    ratings = {"userId": users[rng.integers(0, n_users, n_ratings)], "movieId": ids[rng.integers(0, n, n_ratings)],
               "rating": rng.integers(1, 11, n_ratings) / 2}
    has = rng.random(n) < 0.8
    uhas = rng.random(n_users) < 0.7
    spec = default_spec("neuralcf", n_movies=n + 1, n_users=n_users + 1)
    return ({"movieId": ids, "genres": genres}, ratings,
            (ids[has], rng.standard_normal((int(has.sum()), dim)).astype(np.float32)),
            (users[uhas], rng.standard_normal((int(uhas.sum()), dim)).astype(np.float32)), spec, init_weights(spec, 1))


def run(name, data, warmup, repeats, oracle_users, gpu):
    from oracle import recforyou as R
    from oracle.similar_recall import RecallCatalogue
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.recforyou import RecForYou
    from sparrowrecsys_b200.similar import SimilarMovies, genre_lists
    movies, ratings, emb, uemb, spec, W = data
    users = np.unique(ratings["userId"])
    cat = RecallCatalogue(movies["movieId"], genre_lists(movies["genres"]), ratings["movieId"],
                          np.asarray(ratings["rating"], np.float32), *emb)
    orc = R.RecForYou(cat, ratings["userId"], *uemb)
    score_fn = R.ctr_score_fn(spec, W)
    lines = []
    with SimilarMovies(movies, ratings, emb) as s, RecForYou(s, ratings, uemb) as page, CTRModel(spec, W) as model:
        for ranker in RANKERS:
            t = timed(lambda: page.recommend_arrays(users, SIZE, ranker, model), warmup, repeats)
            orc.rec_list(int(users[0]), SIZE, ranker, score_fn)          # the candidate list, built once
            t0 = time.perf_counter()
            for u in users[:oracle_users].tolist():
                orc.rec_list(u, SIZE, ranker, score_fn)
            cpu_s = time.perf_counter() - t0
            line = {"workload": name, "ranker": ranker, "movies": len(movies["movieId"]),
                    "ratings": int(len(ratings["userId"])), "users": len(users), "size": SIZE, "gpu_call": t,
                    "gpu_users_per_s": len(users) / (t["median_ms"] / 1e3),
                    "oracle_users_timed": min(oracle_users, len(users)),
                    "oracle_users_per_s": min(oracle_users, len(users)) / cpu_s, "gpu": gpu}
            print(json.dumps(line), flush=True)
            lines.append(line)
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-users", type=int, default=300)
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = gpu_info()
    lines = run("reference", reference_data(), a.warmup, a.repeats, a.oracle_users, gpu)
    lines += run("synthetic_30000_users", synthetic_data(), a.warmup, a.repeats, a.oracle_users, gpu)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "recforyou_throughput.jsonl"), "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
