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

Then "nerualcf" with the models that read the uf: / mf: features (DESIGN.md section 4.26): DIN of the reference's
shape and at E = 32 / T = 50, DeepFM, Wide&Deep and EmbeddingMLP, over the golden model samples' hashes (reference)
or seeded hashes for 60 % of the users (synthetic).  Per model: the median of --repeats `recommend` calls over every
user at size 20, against one pass of a Python loop of `CTRModel.rank_user` over the same users - the per-user path,
which was the only way to rank those models per user before the page took them.
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


FEATURE_MODELS = (("din", {}), ("din_e32_t50", {"emb_dim": 32, "hist_len": 50}), ("deepfm", {}),
                  ("widendeep", {}), ("embeddingmlp", {}))


def reference_store():
    from sparrowrecsys_b200 import featurestore as FS
    z = np.load(os.path.join(ROOT, "tests", "golden", "featureeng_model_samples.npz"))
    return FS.FeatureStore.from_samples({k: [str(x) for x in z[k].tolist()] for k in z.files
                                         if z[k].ndim == 1 and k != "text"})


def synthetic_store(users, movie_ids, seed=0):
    from sparrowrecsys_b200 import featurestore as FS
    from sparrowrecsys_b200.spec import GENRE_VOCAB
    rng = np.random.default_rng(seed)
    store = FS.FeatureStore()
    for u in users[rng.random(len(users)) < 0.6].tolist():
        h = {"userRatedMovie%d" % k: str(int(rng.choice(movie_ids))) for k in range(1, 6)}
        h.update({"userGenre%d" % g: GENRE_VOCAB[int(rng.integers(0, len(GENRE_VOCAB)))] for g in range(1, 4)})
        h.update({"userRatingCount": str(int(rng.integers(1, 500))), "userAvgRating": "%.2f" % rng.uniform(1, 5)})
        store.backend.hset("uf:%d" % u, h)
    for m in movie_ids.tolist():
        store.backend.hset("mf:%d" % m, {"movieGenre1": GENRE_VOCAB[m % len(GENRE_VOCAB)],
                                         "movieRatingCount": str(m % 977), "releaseYear": str(1950 + m % 70),
                                         "movieAvgRating": "%.2f" % (1 + (m % 400) / 100)})
    return store


def run_features(name, data, store, warmup, repeats, gpu):
    from sparrowrecsys_b200 import featurestore as FS
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.recforyou import RecForYou
    from sparrowrecsys_b200.similar import SimilarMovies
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    movies, ratings, _, _, ncf_spec, _ = data
    users = np.unique(ratings["userId"])
    fields = {int(u): store.user_features(int(u)) for u in users.tolist()}
    lines = []
    with SimilarMovies(movies, ratings) as s, RecForYou(s, ratings) as page:
        page.set_user_features(store)
        cands = page.recommend_arrays(users[:1], 800, "default")[0][0]
        for model_name, kw in FEATURE_MODELS:
            spec = default_spec(model_name.split("_")[0], n_movies=ncf_spec.n_movies, n_users=ncf_spec.n_users, **kw)
            with CTRModel(spec, init_weights(spec, 1)) as model:
                model.set_movie_table(FS.MovieFeatureTable.from_store(store, spec.n_movies))
                t = timed(lambda: page.recommend_arrays(users, SIZE, "nerualcf", model), warmup, repeats)
                for u in users[:50].tolist():
                    model.rank_user(u, fields[u], cands, SIZE)
                t0 = time.perf_counter()
                for u in users.tolist():
                    model.rank_user(u, fields[u], cands, SIZE)
                loop_s = time.perf_counter() - t0
                line = {"workload": name, "ranker": "nerualcf", "model": model_name, "kernel": model.kernel_name,
                        "users": len(users), "candidates": len(cands), "size": SIZE, "gpu_call": t,
                        "gpu_users_per_s": len(users) / (t["median_ms"] / 1e3), "rank_user_loop_s": loop_s,
                        "rank_user_users_per_s": len(users) / loop_s, "gpu": gpu}
                print(json.dumps(line), flush=True)
                lines.append(line)
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-users", type=int, default=300)
    ap.add_argument("--out")
    ap.add_argument("--features-only", action="store_true", help="only the models that read the uf: / mf: features")
    a = ap.parse_args()
    gpu = gpu_info()
    ref, syn = reference_data(), synthetic_data()
    lines = []
    if not a.features_only:
        lines += run("reference", ref, a.warmup, a.repeats, a.oracle_users, gpu)
        lines += run("synthetic_30000_users", syn, a.warmup, a.repeats, a.oracle_users, gpu)
    lines += run_features("reference", ref, reference_store(), a.warmup, a.repeats, gpu)
    lines += run_features("synthetic_30000_users", syn,
                          synthetic_store(np.unique(syn[1]["userId"]), syn[0]["movieId"]), a.warmup, a.repeats, gpu)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "recforyou_throughput.jsonl"), "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
