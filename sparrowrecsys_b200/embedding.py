"""Train the item2vec movie embeddings and the user embeddings on the GPU.

This is the reference's Spark job `Embedding.scala:27-138`: Spark MLlib's `Word2Vec` (a hierarchical-softmax
skip-gram trained by SGD) over each user's positive ratings gives `item2vecEmb.csv`, and the sum of those vectors over
each user's ratings gives `userEmb.csv` - the two files the "emb" ranker (`ranking.rank_by_embedding`) reads.
DESIGN.md section 4.12 gives the semantics and the orders Spark leaves open; `oracle/item2vec.py` restates them.

* `item2vec` trains on one device (`srs_item2vec_host`) and returns the vocabulary ids and their vectors.
* `user_embeddings` sums them per user on one device (`srs_user_embeddings_host`).
* `find_synonyms` is Word2VecModel.findSynonyms on the device's cosine scorer and top-k.
* `write_embeddings_csv` writes the reference's text; `ranking.load_embeddings_csv` reads it back.

The rest of the job (`:140-266`, DESIGN.md section 4.14; `oracle/graphemb.py` and `oracle/lsh.py` restate it):

* `item_transitions` and `random_walks` are DeepWalk's transition matrix and walks (`srs_item_transitions_host`,
  `srs_random_walks_host`); `graph_embedding` trains the same Word2Vec on the walks (`srs_graph_embedding_host`).
* `BucketedRandomProjectionLSH(...).fit(vectors)` gives a model whose `transform`, `approx_nearest_neighbors` and
  `approx_similarity_join` run on the device (`srs_lsh_transform_host`, `srs_lsh_query_host`,
  `srs_lsh_similarity_join_host`).

    python -m sparrowrecsys_b200.embedding ratings.csv OUTDIR     # OUTDIR/item2vecEmb.csv, OUTDIR/userEmb.csv
    python -m sparrowrecsys_b200.embedding ratings.csv OUTDIR --graph --lsh   # also itemGraphEmb.csv, the LSH demo
"""
from __future__ import annotations

import ctypes as C
import math
import os
import sys
from typing import Mapping, Tuple

import numpy as np

from . import _lib


def _ratings(ratings: Mapping[str, np.ndarray]):
    user = np.ascontiguousarray(ratings["userId"], np.int32)
    movie = np.ascontiguousarray(ratings["movieId"], np.int32)
    n = user.shape[0]
    if movie.shape[0] != n:
        raise ValueError("ratings columns differ in length")
    return user, movie, n


def _rated(ratings: Mapping[str, np.ndarray]):
    """(user, movie, half-stars int8, timestamp, n) of full ratings, checked."""
    user, movie, n = _ratings(ratings)
    ts = np.ascontiguousarray(ratings["timestamp"], np.int32)
    r2 = np.asarray(ratings["rating"], np.float64) * 2
    if ts.shape[0] != n or r2.shape[0] != n:
        raise ValueError("ratings columns differ in length")
    if not np.array_equal(r2, np.trunc(r2)) or (n and (r2.min() < 1 or r2.max() > 10)):
        raise ValueError("ratings must be half-stars in [0.5, 5]")
    return user, movie, np.ascontiguousarray(r2, np.int8), ts, n


def item2vec(ratings: Mapping[str, np.ndarray], vector_size: int = 10, window_size: int = 5,
             num_iterations: int = 10, num_partitions: int = 1, seed: int = 0, device: int = 0
             ) -> Tuple[np.ndarray, np.ndarray]:
    """Word2Vec.fit over the positive ratings of `ratings` (userId, movieId, rating, timestamp; as
    `featureeng.load_ratings_csv` returns), on `device`.  Returns (ids int32 [V] in vocabulary order - positive
    count descending, ties by id - and vectors float32 [V][vector_size]).  The same inputs give the same bits."""
    user, movie, half, ts, n = _rated(ratings)
    cap = max(1, int(np.unique(movie[half >= 7]).size))
    ids = np.zeros(cap, np.int32)
    vec = np.zeros((cap, int(vector_size)), np.float32)
    params = _lib.SrsItem2vecParams(int(vector_size), int(window_size), int(num_iterations), int(num_partitions),
                                    int(seed) & ((1 << 64) - 1))
    V = C.c_int32(0)
    p = lambda a: a.ctypes.data
    _lib.check(_lib.load().srs_item2vec_host(p(user), p(movie), p(half), p(ts), n, C.byref(params), device, cap,
                                             p(ids), p(vec), C.byref(V)))
    return ids[:V.value].copy(), vec[:V.value].copy()


def user_embeddings(ratings: Mapping[str, np.ndarray], ids, vectors, device: int = 0
                    ) -> Tuple[np.ndarray, np.ndarray]:
    """Per user (ascending) the float32 sum of the vectors of every movie the user rated (any rating) that has one,
    in reverse ratings order, with no division - as the reference's shipped userEmb.csv was made.  Returns
    (user ids int32 [U], vectors float32 [U][dim])."""
    user, movie, n = _ratings(ratings)
    ids = np.ascontiguousarray(ids, np.int32)
    vectors = np.ascontiguousarray(vectors, np.float32)
    if vectors.ndim != 2 or vectors.shape[0] != ids.shape[0]:
        raise ValueError("ids [n] and vectors [n, dim] expected")
    D = vectors.shape[1]
    cap = max(1, int(np.unique(user).size))
    uids = np.zeros(cap, np.int32)
    out = np.zeros((cap, D), np.float32)
    U = C.c_int32(0)
    p = lambda a: a.ctypes.data
    _lib.check(_lib.load().srs_user_embeddings_host(p(user), p(movie), n, p(ids), p(vectors), ids.shape[0], D, device,
                                                    cap, p(uids), p(out), C.byref(U)))
    return uids[:U.value].copy(), out[:U.value].copy()


def find_synonyms(ids, vectors, movie_id: int, num: int, device: int = 0):
    """Word2VecModel.findSynonyms(movie_id, num) (Embedding.scala:112): the `num` movies of highest cosine
    similarity to `movie_id`'s vector, best first, the movie itself excluded.  Returns (ids int32, similarities
    float32).  KeyError if the movie has no vector."""
    from .ranking import rank_by_embedding
    ids = np.asarray(ids, np.int32)
    where = np.flatnonzero(ids == int(movie_id))
    if where.size == 0:
        raise KeyError("movie %d has no vector" % movie_id)
    vectors = np.ascontiguousarray(vectors, np.float32)
    pos, sim = rank_by_embedding(vectors[where[0]], vectors, int(num) + 1, device)
    keep = pos != where[0]
    return ids[pos[keep]][:num], sim[keep][:num]


MAX_WALK_WORDS = 21000000          # num_walks * walk_length: the library's bound on the walk corpus


def item_transitions(ratings: Mapping[str, np.ndarray], device: int = 0) -> dict:
    """generateTransitionMatrix over the positive sentences, on `device`.  Returns a dict: sources int32 [S]
    ascending, out int32 [S] (pairs leaving each source), dist float64 [S] (out / pairTotal), row_ptr int32 [S + 1],
    and per pair, by source then target ascending, targets int32 [E], counts int32 [E], probs float64 [E]
    (count / out of its source)."""
    user, movie, half, ts, n = _rated(ratings)
    pos = half >= 7
    s_cap = max(1, int(np.unique(movie[pos]).size))
    e_cap = max(1, int(pos.sum()))
    src, rp, out, dist = (np.zeros(s_cap, np.int32), np.zeros(s_cap + 1, np.int32), np.zeros(s_cap, np.int32),
                          np.zeros(s_cap, np.float64))
    tgt, cnt, prob = np.zeros(e_cap, np.int32), np.zeros(e_cap, np.int32), np.zeros(e_cap, np.float64)
    S, E = C.c_int32(0), C.c_int32(0)
    p = lambda a: a.ctypes.data
    _lib.check(_lib.load().srs_item_transitions_host(p(user), p(movie), p(half), p(ts), n, device, s_cap, e_cap,
                                                     p(src), p(rp), p(out), p(dist), p(tgt), p(cnt), p(prob),
                                                     C.byref(S), C.byref(E)))
    S, E = S.value, E.value
    return {"sources": src[:S].copy(), "out": out[:S].copy(), "dist": dist[:S].copy(), "row_ptr": rp[:S + 1].copy(),
            "targets": tgt[:E].copy(), "counts": cnt[:E].copy(), "probs": prob[:E].copy()}


def _check_walks(num_walks, walk_length):
    W, L = int(num_walks), int(walk_length)
    if W < 1 or L < 1 or W * L > MAX_WALK_WORDS:
        raise ValueError("%d walks of length %d: both must be >= 1 and their product <= %d"
                         % (W, L, MAX_WALK_WORDS))
    return W, L


def random_walks(ratings: Mapping[str, np.ndarray], num_walks: int = 20000, walk_length: int = 10, seed: int = 0,
                 device: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """randomWalk (Embedding.scala:140-184) over `item_transitions`, on `device`: (walks int32 [num_walks]
    [walk_length], -1 past each walk's end, and lengths int32 [num_walks]).  A walk stops at a movie with no
    outgoing pair; DESIGN.md section 4.14 gives the draws.  The same inputs give the same walks."""
    user, movie, half, ts, n = _rated(ratings)
    W, L = _check_walks(num_walks, walk_length)
    walks = np.zeros((W, L), np.int32)
    lengths = np.zeros(W, np.int32)
    p = lambda a: a.ctypes.data
    _lib.check(_lib.load().srs_random_walks_host(p(user), p(movie), p(half), p(ts), n, W, L,
                                                 int(seed) & ((1 << 64) - 1), device, p(walks), p(lengths)))
    return walks, lengths


def graph_embedding(ratings: Mapping[str, np.ndarray], vector_size: int = 10, window_size: int = 5,
                    num_iterations: int = 10, num_partitions: int = 1, seed: int = 0, num_walks: int = 20000,
                    walk_length: int = 10, device: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """graphEmb (Embedding.scala:254-266): `random_walks(ratings, num_walks, walk_length, seed)`, each non-empty
    walk one sentence, trained by `item2vec`'s Word2Vec with the same arguments and seed.  Returns (ids int32 [V],
    vectors float32 [V][vector_size]) as `item2vec` does."""
    user, movie, half, ts, n = _rated(ratings)
    W, L = _check_walks(num_walks, walk_length)
    cap = max(1, min(int(np.unique(movie[half >= 7]).size), W * L // 5))
    ids = np.zeros(cap, np.int32)
    vec = np.zeros((cap, int(vector_size)), np.float32)
    params = _lib.SrsItem2vecParams(int(vector_size), int(window_size), int(num_iterations), int(num_partitions),
                                    int(seed) & ((1 << 64) - 1))
    V = C.c_int32(0)
    p = lambda a: a.ctypes.data
    _lib.check(_lib.load().srs_graph_embedding_host(p(user), p(movie), p(half), p(ts), n, C.byref(params), W, L,
                                                    device, cap, p(ids), p(vec), C.byref(V)))
    return ids[:V.value].copy(), vec[:V.value].copy()


# ---- BucketedRandomProjectionLSH (Embedding.scala:230-252) -------------------------------------------------------

class _JavaRandom:
    """java.util.Random: the 48-bit linear congruential generator and the polar nextGaussian its javadoc specifies."""

    def __init__(self, seed: int):
        self._s = (int(seed) ^ 0x5DEECE66D) & ((1 << 48) - 1)
        self._cached = None

    def _next(self, bits: int) -> int:
        self._s = (self._s * 0x5DEECE66D + 0xB) & ((1 << 48) - 1)
        return self._s >> (48 - bits)

    def next_double(self) -> float:
        return ((self._next(26) << 27) + self._next(27)) * 2.0 ** -53

    def next_gaussian(self) -> float:
        if self._cached is not None:
            g, self._cached = self._cached, None
            return g
        while True:
            v1, v2 = 2 * self.next_double() - 1, 2 * self.next_double() - 1
            s = v1 * v1 + v2 * v2
            if 0 < s < 1:
                break
        m = math.sqrt(-2 * math.log(s) / s)
        self._cached = v2 * m
        return v1 * m


LSH_DEFAULT_SEED = 772209414      # "org.apache.spark.ml.feature.BucketedRandomProjectionLSH".hashCode (HasSeed)
LSH_MAX_K = 256


class BucketedRandomProjectionLSH:
    """Spark ML's BucketedRandomProjectionLSH estimator: `fit(vectors)` draws `num_hash_tables` unit vectors of the
    vectors' dimension from java.util.Random(seed) (Gaussians divided by their L2 norm)."""

    def __init__(self, bucket_length: float = 0.1, num_hash_tables: int = 3, seed: int = LSH_DEFAULT_SEED):
        if not (math.isfinite(bucket_length) and bucket_length > 0):
            raise ValueError("bucket_length must be finite and > 0")
        if int(num_hash_tables) < 1:
            raise ValueError("num_hash_tables must be >= 1")
        self.bucket_length = float(bucket_length)
        self.num_hash_tables = int(num_hash_tables)
        self.seed = int(seed)

    def fit(self, vectors) -> "BucketedRandomProjectionLSHModel":
        dim = np.asarray(vectors).shape[-1]
        rand = _JavaRandom(self.seed)
        uv = np.zeros((self.num_hash_tables, dim))
        for j in range(self.num_hash_tables):
            g = [rand.next_gaussian() for _ in range(dim)]
            sq = 0.0
            for x in g:
                sq = sq + x * x
            norm = math.sqrt(sq)
            uv[j] = [x / norm for x in g]
        return BucketedRandomProjectionLSHModel(uv, self.bucket_length)


def _float32_rows(vectors, dim):
    v = np.asarray(vectors)
    v32 = np.ascontiguousarray(v, np.float32)
    if v32.ndim != 2 or v32.shape[1] != dim:
        raise ValueError("vectors [n, %d] expected, got shape %s" % (dim, v.shape))
    if not np.array_equal(v32.astype(np.float64), v.astype(np.float64)):
        raise ValueError("vectors must be float32 values (the item vectors are)")
    if not np.all(np.isfinite(v32)):
        raise ValueError("vectors must be finite")
    return v32


class BucketedRandomProjectionLSHModel:
    """`rand_unit_vectors` [num_hash_tables][dim] float64 and `bucket_length`; hashing and queries run on the
    device."""

    def __init__(self, rand_unit_vectors, bucket_length: float):
        self.rand_unit_vectors = np.ascontiguousarray(rand_unit_vectors, np.float64)
        self.bucket_length = float(bucket_length)
        if self.rand_unit_vectors.ndim != 2 or not np.all(np.isfinite(self.rand_unit_vectors)):
            raise ValueError("rand_unit_vectors must be a finite [tables, dim] array")

    @property
    def dim(self) -> int:
        return self.rand_unit_vectors.shape[1]

    def transform(self, vectors, device: int = 0) -> np.ndarray:
        """Bucket ids float64 [n][num_hash_tables]: floor(dot(x, v_j) / bucket_length) of the float32 vectors."""
        x = _float32_rows(vectors, self.dim)
        out = np.zeros((x.shape[0], self.rand_unit_vectors.shape[0]), np.float64)
        _lib.check(_lib.load().srs_lsh_transform_host(x.ctypes.data, x.shape[0], self.dim,
                                                      self.rand_unit_vectors.ctypes.data,
                                                      self.rand_unit_vectors.shape[0], self.bucket_length, device,
                                                      out.ctypes.data))
        return out

    def approx_nearest_neighbors(self, ids, vectors, keys, k: int, device: int = 0):
        """approxNearestNeighbors(dataset, key, k), single probe: the rows sharing a key's bucket in at least one
        table, by Euclidean distance ascending (ties by id), at most k.  `keys` [dim] gives (ids int32, distances
        float64); [Q][dim] gives a list of Q such pairs, computed in one device call."""
        x = _float32_rows(vectors, self.dim)
        ids = np.ascontiguousarray(ids, np.int32)
        if ids.shape != (x.shape[0],):
            raise ValueError("ids [n] expected for %d vectors" % x.shape[0])
        q = np.ascontiguousarray(keys, np.float64)
        single = q.ndim == 1
        q = q.reshape(1, -1) if single else q
        if q.ndim != 2 or q.shape[1] != self.dim:
            raise ValueError("keys [%d] or [Q, %d] expected, got shape %s" % (self.dim, self.dim, np.shape(keys)))
        if not np.all(np.isfinite(q)):
            raise ValueError("keys must be finite")
        if not 1 <= int(k) <= LSH_MAX_K:
            raise ValueError("k must be in 1..%d" % LSH_MAX_K)
        k = int(k)
        Q = q.shape[0]
        oid = np.zeros((max(Q, 1), k), np.int32)
        odist = np.zeros((max(Q, 1), k), np.float64)
        ocnt = np.zeros(max(Q, 1), np.int32)
        _lib.check(_lib.load().srs_lsh_query_host(ids.ctypes.data, x.ctypes.data, x.shape[0], self.dim,
                                                  self.rand_unit_vectors.ctypes.data,
                                                  self.rand_unit_vectors.shape[0], self.bucket_length,
                                                  q.ctypes.data, Q, k, device, oid.ctypes.data, odist.ctypes.data,
                                                  ocnt.ctypes.data))
        res = [(oid[i, :ocnt[i]].copy(), odist[i, :ocnt[i]].copy()) for i in range(Q)]
        return res[0] if single else res

    def approx_similarity_join(self, ids_a, vectors_a, ids_b, vectors_b, threshold: float, device: int = 0):
        """approxSimilarityJoin(datasetA, datasetB, threshold): every pair (a, b) sharing a bucket in at least one
        table, once, with Euclidean distance < threshold, ordered by (id_a, id_b).  Ids must be unique within each
        side; pass the same arrays twice for a self-join.  Returns (ids_a int32 [P], ids_b int32 [P], distances
        float64 [P]), computed on the device."""
        sides = []
        for name, ids, vectors in (("a", ids_a, vectors_a), ("b", ids_b, vectors_b)):
            x = _float32_rows(vectors, self.dim)
            ids = np.ascontiguousarray(ids, np.int32)
            if ids.shape != (x.shape[0],):
                raise ValueError("ids_%s [n] expected for %d vectors" % (name, x.shape[0]))
            u, counts = np.unique(ids, return_counts=True)
            if np.any(counts > 1):
                raise ValueError("ids_%s holds id %d more than once" % (name, u[np.argmax(counts > 1)]))
            sides.append((ids, x))
        (ia, xa), (ib, xb) = sides
        fn = _lib.load().srs_lsh_similarity_join_host
        P = C.c_int64(0)
        capacity = min(len(ia) * len(ib), 1 << 20)
        for _ in range(2):                       # a first guess at the size, then the size the library reported
            oa, ob = np.zeros(max(capacity, 1), np.int32), np.zeros(max(capacity, 1), np.int32)
            od = np.zeros(max(capacity, 1), np.float64)
            rc = fn(ia.ctypes.data, xa.ctypes.data, len(ia), ib.ctypes.data, xb.ctypes.data, len(ib), self.dim,
                    self.rand_unit_vectors.ctypes.data, self.rand_unit_vectors.shape[0], self.bucket_length,
                    float(threshold), device, capacity, oa.ctypes.data, ob.ctypes.data, od.ctypes.data,
                    C.byref(P))
            if rc != _lib.SRS_ERR_RANGE:
                break
            capacity = P.value
        _lib.check(rc)
        n = P.value
        return oa[:n].copy(), ob[:n].copy(), od[:n].copy()


# the reference's sample key (Embedding.scala:250)
LSH_SAMPLE_KEY = np.array([0.795, 0.583, 1.120, 0.850, 0.174, -0.839, -0.0633, 0.249, 0.673, -0.237])


def print_lsh_demo(ids, vectors, device: int = 0) -> None:
    """embeddingLSH's output: the bucket ids of the first 10 movies in vocabulary order, and the 5 approximate
    nearest neighbours of the reference's sample key (vectors of dimension 10)."""
    model = BucketedRandomProjectionLSH().fit(vectors)
    buckets = model.transform(np.asarray(vectors)[:10], device)
    print("movieId, bucketId of the first 10 movies:")
    for i, b in zip(np.asarray(ids)[:10].tolist(), buckets.tolist()):
        print(i, "[" + ",".join(repr(x) for x in b) + "]")
    print("Approximately searching for 5 nearest neighbors of the sample embedding:")
    nid, nd = model.approx_nearest_neighbors(ids, vectors, LSH_SAMPLE_KEY, 5, device)
    for i, d in zip(nid.tolist(), nd.tolist()):
        print(i, repr(d))


def java_float_string(x) -> str:
    """java.lang.Float.toString: the shortest digits that round-trip to the float32, plain for 1e-3 <= |x| < 1e7
    (at least one digit after the point), otherwise d.ddd...E<exponent>."""
    x = np.float32(x)
    if x == 0:
        return "-0.0" if np.signbit(x) else "0.0"
    if not np.isfinite(x):
        return "NaN" if np.isnan(x) else ("Infinity" if x > 0 else "-Infinity")
    s = np.format_float_scientific(x, unique=True, trim="-")
    sign = "-" if s[0] == "-" else ""
    mant, exp = s.lstrip("-").split("e")
    digits = mant.replace(".", "")
    e = int(exp)
    if 1e-3 <= abs(float(x)) < 1e7:
        if e >= 0:
            head = digits[:e + 1].ljust(e + 1, "0")
            tail = digits[e + 1:] or "0"
        else:
            head, tail = "0", "0" * (-e - 1) + digits
        return "%s%s.%s" % (sign, head, tail)
    return "%s%s.%sE%d" % (sign, digits[0], digits[1:] or "0", e)


def write_embeddings_csv(path: str, ids, vectors) -> None:
    """The reference's embedding text (Embedding.scala:118-122, 85-88): one `id:v v v ...` line per row, each
    value as Java's Float.toString prints it."""
    vectors = np.asarray(vectors, np.float32)
    with open(path, "w", newline="") as f:
        for i, row in zip(np.asarray(ids).tolist(), vectors):
            f.write("%d:%s\n" % (i, " ".join(java_float_string(v) for v in row)))


def _print_synonyms(ids, vec):
    sids, sim = find_synonyms(ids, vec, 158, 20) if 158 in ids else ((), ())
    for s, c in zip(np.asarray(sids).tolist(), np.asarray(sim).tolist()):
        print(s, c)


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    flags = {a for a in argv if a.startswith("--")}
    argv = [a for a in argv if not a.startswith("--")]
    if len(argv) != 2 or flags - {"--graph", "--lsh"}:
        sys.stderr.write("usage: python -m sparrowrecsys_b200.embedding ratings.csv OUTDIR [--graph] [--lsh]\n")
        return 2
    from .featureeng import load_ratings_csv
    ratings = load_ratings_csv(argv[0])
    os.makedirs(argv[1], exist_ok=True)
    ids, vec = item2vec(ratings)
    _print_synonyms(ids, vec)
    write_embeddings_csv(os.path.join(argv[1], "item2vecEmb.csv"), ids, vec)
    if "--lsh" in flags:
        print_lsh_demo(ids, vec)
    if "--graph" in flags:                               # graphEmb, as if Embedding.scala:283 ran
        gids, gvec = graph_embedding(ratings)
        _print_synonyms(gids, gvec)
        write_embeddings_csv(os.path.join(argv[1], "itemGraphEmb.csv"), gids, gvec)
        if "--lsh" in flags:
            print_lsh_demo(gids, gvec)
    uids, uvec = user_embeddings(ratings, ids, vec)
    write_embeddings_csv(os.path.join(argv[1], "userEmb.csv"), uids, uvec)
    return 0


if __name__ == "__main__":
    sys.exit(main())
