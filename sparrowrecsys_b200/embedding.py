"""Train the item2vec movie embeddings and the user embeddings on the GPU.

This is the reference's Spark job `Embedding.scala:27-138`: Spark MLlib's `Word2Vec` (a hierarchical-softmax
skip-gram trained by SGD) over each user's positive ratings gives `item2vecEmb.csv`, and the sum of those vectors over
each user's ratings gives `userEmb.csv` - the two files the "emb" ranker (`ranking.rank_by_embedding`) reads.
DESIGN.md section 4.12 gives the semantics and the orders Spark leaves open; `oracle/item2vec.py` restates them.

* `item2vec` trains on one device (`srs_item2vec_host`) and returns the vocabulary ids and their vectors.
* `user_embeddings` sums them per user on one device (`srs_user_embeddings_host`).
* `find_synonyms` is Word2VecModel.findSynonyms on the device's cosine scorer and top-k.
* `write_embeddings_csv` writes the reference's text; `ranking.load_embeddings_csv` reads it back.

    python -m sparrowrecsys_b200.embedding ratings.csv OUTDIR     # OUTDIR/item2vecEmb.csv, OUTDIR/userEmb.csv
"""
from __future__ import annotations

import ctypes as C
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


def item2vec(ratings: Mapping[str, np.ndarray], vector_size: int = 10, window_size: int = 5,
             num_iterations: int = 10, num_partitions: int = 1, seed: int = 0, device: int = 0
             ) -> Tuple[np.ndarray, np.ndarray]:
    """Word2Vec.fit over the positive ratings of `ratings` (userId, movieId, rating, timestamp; as
    `featureeng.load_ratings_csv` returns), on `device`.  Returns (ids int32 [V] in vocabulary order - positive
    count descending, ties by id - and vectors float32 [V][vector_size]).  The same inputs give the same bits."""
    user, movie, n = _ratings(ratings)
    ts = np.ascontiguousarray(ratings["timestamp"], np.int32)
    r2 = np.asarray(ratings["rating"], np.float64) * 2
    if ts.shape[0] != n or r2.shape[0] != n:
        raise ValueError("ratings columns differ in length")
    if not np.array_equal(r2, np.trunc(r2)) or (n and (r2.min() < 1 or r2.max() > 10)):
        raise ValueError("ratings must be half-stars in [0.5, 5]")
    half = np.ascontiguousarray(r2, np.int8)
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


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) != 2:
        sys.stderr.write("usage: python -m sparrowrecsys_b200.embedding ratings.csv OUTDIR\n")
        return 2
    from .featureeng import load_ratings_csv
    ratings = load_ratings_csv(argv[0])
    os.makedirs(argv[1], exist_ok=True)
    ids, vec = item2vec(ratings)
    sids, sim = find_synonyms(ids, vec, 158, 20) if 158 in ids else ((), ())
    for s, c in zip(np.asarray(sids).tolist(), np.asarray(sim).tolist()):
        print(s, c)
    write_embeddings_csv(os.path.join(argv[1], "item2vecEmb.csv"), ids, vec)
    uids, uvec = user_embeddings(ratings, ids, vec)
    write_embeddings_csv(os.path.join(argv[1], "userEmb.csv"), uids, uvec)
    return 0


if __name__ == "__main__":
    sys.exit(main())
