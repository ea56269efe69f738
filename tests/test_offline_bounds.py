"""The offline jobs at their bounds and tile edges (csrc/item2vec.cu, graphemb.cu, lsh.cu with the similarity join,
als.cu with implicit ALS, RankingMetrics and nonnegative ALS, featureeng.cu, featurejob.cu, binary_metrics.cu, and
hostcall.h's grid cap).

`BOUNDS` names one case per (job, edge).  Each case builds its inputs here; its `reach` shows from the oracle alone,
with no device, that the inputs reach the edge the case names, and returns the (bound, value) pairs it reaches.
tests/test_gpu_offline_bounds.py runs every case on the device against its oracle, bit for bit, twice.

The bounds come from the kernels' own constants: `test_every_bound_has_a_case` parses them, so a changed constant
without a case at its new value fails.  The size bounds (21 000 000 ratings, kMaxWalkWords, featurejob.cu's
kMaxValues) are covered by the rejection one past them; the deepest Huffman case is the largest run of the first
jobs, and featurejob.cu's rating features run at 21 000 000 ratings and its StringIndexer at kMaxTokens.
"""
from __future__ import annotations

import ctypes as C
import functools
import math
import os
import re
from typing import Callable, NamedTuple

import numpy as np
import pytest

from oracle import als as A
from oracle import als_implicit as XP
from oracle import als_nnls as N
from oracle import binary_metrics as BM
from oracle import feature_job as FQ
from oracle import feature_eng as F
from oracle import graphemb as G
from oracle import item2vec as I
from oracle import lsh as H
from sparrowrecsys_b200 import _lib

from test_item2vec_oracle import MAX_RATINGS, _deepest_counts

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc")


# ---- the kernels' constants --------------------------------------------------------------------------------------
def constants(*files):
    """name -> value of every `constexpr` integer in the given csrc files (simple integer expressions).  A name
    defined in two files with two values raises ValueError rather than letting the last file win."""
    out = {}
    for f in files:
        with open(os.path.join(CSRC, f)) as fh:
            src = fh.read()
        for name, expr in re.findall(r"constexpr\s+(?:unsigned|int|int32_t|int64_t|uint32_t|uint64_t)\s+(k\w+)\s*="
                                     r"\s*([^;]+);", src):
            e = re.sub(r"(?<=\d)(?:ULL|ull|LL|u|U)\b", "", expr)
            for k in sorted(out, key=len, reverse=True):
                e = re.sub(r"\b%s\b" % k, str(out[k]), e)
            try:
                v = int(eval(e, {"__builtins__": {}}))
            except (NameError, SyntaxError):
                continue
            if name in out and out[name] != v:
                raise ValueError("%s is %d in %s but %d in an earlier file" % (name, v, f, out[name]))
            out[name] = v
    return out


RATING_BOUND_FILES = ("als.cu", "featureeng.cu", "item2vec.cu", "featurejob.cu")
K = constants("als.cu", "lsh.cu", "item2vec.cu", "featureeng.cu", "graphemb.cu", "featurejob.cu", "hostcall.h")
KB = constants("binary_metrics.cu", "hostcall.h")     # its own table: its kChunk (points) is not als.cu's (ratings)


class Case(NamedTuple):
    job: str
    make: Callable[[], dict]
    reach: Callable[[dict], set]


# ---- item2vec and DeepWalk ---------------------------------------------------------------------------------------
def _ratings_of_sentences(sentences, first_user=1):
    """Each sentence one user's positive ratings (4.0), timestamps 10 digits in sentence order."""
    lens = np.array([len(s) for s in sentences], np.int64)
    movie = np.concatenate(sentences).astype(np.int32)
    user = np.repeat(np.arange(first_user, first_user + len(sentences)), lens).astype(np.int32)
    pos = np.arange(len(movie)) - np.repeat(np.r_[0, np.cumsum(lens)[:-1]], lens)
    return {"userId": user, "movieId": movie, "rating": np.full(len(movie), 4.0),
            "timestamp": (1000000000 + pos).astype(np.int32)}


def corpus(seqs, ids, max_len=I.MAX_SENTENCE_LENGTH):
    """I.chunk_corpus, vectorised for the large corpora: (words int32, offsets int64)."""
    lens = np.array([len(s) for s in seqs], np.int64)
    allw = np.concatenate(seqs).astype(np.int64)
    sid = np.repeat(np.arange(len(seqs)), lens)
    o = np.argsort(ids, kind="stable")
    j = np.minimum(np.searchsorted(ids[o], allw), len(ids) - 1)
    found = ids[o][j] == allw
    w, s = o[j[found]].astype(np.int32), sid[found]
    first = np.r_[True, s[1:] != s[:-1]]
    start = np.maximum.accumulate(np.where(first, np.arange(len(s)), 0))
    cut = (np.arange(len(s)) - start) % max_len == 0
    return w, np.r_[np.flatnonzero(cut), len(w)].astype(np.int64)


def _caterpillar(depth, D, window, P, seed):
    """The smallest corpus with a Huffman code of `depth` (_deepest_counts), shuffled into sentences of 1000."""
    counts = np.array(_deepest_counts(depth), np.int64)
    ids = 100 + np.arange(len(counts))
    words = np.repeat(ids, counts)
    np.random.default_rng(depth).shuffle(words)
    sents = np.split(words, np.arange(1000, len(words), 1000))
    return dict(ratings=_ratings_of_sentences(sents), seqs=sents, depth=depth,
                params=dict(vector_size=D, window_size=window, num_iterations=1, num_partitions=P, seed=seed))


def _sentence_edges():
    """Users of exactly 1000 and 1001 words (the second cut into 1000 + 1), and users shorter than the window."""
    rng = np.random.default_rng(12)
    vocab = np.arange(7, 37)
    lens = [1000, 1001, 1, 2, 3, 999]
    sents = [rng.choice(vocab, n) for n in lens]
    sents[2] = np.array([7])
    return dict(ratings=_ratings_of_sentences(sents), seqs=sents, depth=None,
                params=dict(vector_size=33, window_size=1200, num_iterations=2, num_partitions=1, seed=3))


def i2v_oracle_input(d):
    ids, counts = I.build_vocab(d["seqs"])
    words, offs = corpus(d["seqs"], ids)
    code, point, codelen = I.huffman(counts)
    return ids, counts, words, offs, code, point, codelen


def _i2v_reach(d):
    ids, counts, words, offs, code, point, codelen = i2v_oracle_input(d)
    p = d["params"]
    got = {("kMaxDim", p["vector_size"]), ("partitions", p["num_partitions"])}
    sl = np.diff(offs)
    if d["depth"] is not None:
        assert codelen.max() == d["depth"], codelen.max()
        assert sl.max() <= I.MAX_SENTENCE_LENGTH
        got.add(("kMaxCode", int(codelen.max())))
    else:
        assert 1000 in sl.tolist() and 1 in sl.tolist()                # 1000 words, and the 1001st on its own
        assert {1000, 1001} <= {len(s) for s in d["seqs"]}
        assert p["window_size"] > max(len(s) for s in d["seqs"])        # the window is longer than any sentence
        ref_w, ref_o = I.chunk_corpus(d["seqs"], ids)
        assert np.array_equal(ref_w, words) and np.array_equal(ref_o, offs)
        got |= {("sentence", 1000), ("sentence", 1001), ("window>sentence", 1)}
    return got


DEEPEST = max(d for d in range(2, 40) if sum(_deepest_counts(d)) <= MAX_RATINGS)   # 31


def _hub_depth_graph():
    """One source (a hub) whose 25 targets' pair counts grow by 1.66: 3 000 000 walks of length 2 give walk words
    whose Huffman tree is a caterpillar at least 24 deep."""
    hub = K["kIdMask"] - 2
    c = np.round(1.66 ** np.arange(25)).astype(np.int64)[::-1]
    targets = np.arange(25) + 100
    sents = [np.array([hub, t]) for t, n in zip(targets.tolist(), c.tolist()) for _ in range(n)]
    return dict(ratings=_ratings_of_sentences(sents), walks=[(3000000, 2)], min_depth=24,
                params=dict(vector_size=10, window_size=5, num_iterations=1, num_partitions=64, seed=0))


def _top_id_hub_graph():
    """Ids 2^24 - 1 and 2^24 - 2 as sources and targets, and a hub row with 5 000 targets."""
    top = K["kIdMask"]
    hub = top - 1
    rng = np.random.default_rng(4)
    sents = [np.array([hub, t]) for t in np.r_[np.arange(1, 5000), top].tolist()]
    sents += [np.array([top, hub, top, 3, hub, top - 5]) for _ in range(20)]
    sents += [rng.choice(np.r_[1, 2, 3, hub, top], 12) for _ in range(300)]
    return dict(ratings=_ratings_of_sentences(sents), walks=[(20000, 1), (20000, 2), (20000, 10)], min_depth=None,
                params=dict(vector_size=8, window_size=5, num_iterations=1, num_partitions=1, seed=5))


def graph_transitions(d):
    r = d["ratings"]
    _, seqs = I.positive_sequences(r["userId"], r["movieId"], np.rint(r["rating"] * 2), r["timestamp"])
    return G.transitions(seqs)


def _graph_reach(d):
    tr = graph_transitions(d)
    got = {("walk_length", L) for _, L in d["walks"]}
    rows = np.diff(tr["row_ptr"])
    if d["min_depth"] is not None:
        W, L = d["walks"][0]
        w, n = G.random_walks(tr, W, L, seed=d["params"]["seed"])
        ids, cnt = np.unique(w[w >= 0], return_counts=True)
        keep = cnt >= I.MIN_COUNT
        codelen = I.huffman(np.sort(cnt[keep])[::-1])[2]
        assert codelen.max() >= d["min_depth"], codelen.max()
        got.add(("walk_depth", int(codelen.max())))
    else:
        top = K["kIdMask"]
        assert {top, top - 1} <= set(tr["sources"].tolist())
        assert {top, top - 1} <= set(tr["targets"].tolist())
        assert rows.max() >= 5000
        got |= {("kIdMask", top), ("kIdMask", top - 1), ("hub_row", int(rows.max()))}
    return got


# ---- LSH --------------------------------------------------------------------------------------------------------
def _nonneg_unit(D, L, seed):
    v = np.abs(H.fit(D, L, seed=seed))
    return v / np.sqrt((v * v).sum(axis=1, keepdims=True))


def _lsh_full():
    """Every row a candidate (nonnegative rows and unit vectors, bucket length 1e6: every bucket id 0), 20 000 rows:
    each warp's list fills.  Rows 7 + 32 j (eight warps) are one vector, half with one id and half with distinct
    ids, so ties are broken by id and then by row across warps."""
    rng = np.random.default_rng(21)
    n, D, L = 20000, 16, 3
    x = rng.random((n, D)).astype(np.float32)
    ids = rng.permutation(10 * n)[:n].astype(np.int32)
    dup = 7 + 32 * np.arange(16)
    x[dup] = x[7]
    ids[dup[:8]] = ids[7]
    ids[dup[8:]] = 3 + np.arange(8)[::-1]
    keys = np.r_[x[[7, 0, 5000]].astype(np.float64), rng.random((2, D))]
    return dict(ids=ids, x=x, uv=_nonneg_unit(D, L, 8), bl=1e6, keys=keys, ks=[1, 255, 256], dup=dup)


def _lsh_small():
    rng = np.random.default_rng(22)
    n, D, L = 100, 8, 2
    x = rng.standard_normal((n, D)).astype(np.float32)
    return dict(ids=np.arange(n, dtype=np.int32) * 5, x=x, uv=H.fit(D, L, seed=3), bl=4.0,
                keys=np.r_[x[:3].astype(np.float64), rng.standard_normal((2, D))], ks=[1, 256], dup=None)


def _lsh_wide(D, L, n, bl):
    rng = np.random.default_rng(D + L)
    x = rng.standard_normal((n, D)).astype(np.float32)
    x[11] = x[10]
    return dict(ids=rng.permutation(4 * n)[:n].astype(np.int32), x=x, uv=H.fit(D, L, seed=D), bl=bl,
                keys=np.r_[x[[10, 0, 1]].astype(np.float64), rng.standard_normal((2, D))], ks=[7, 256], dup=None)


def _lsh_reach(d):
    x, uv, bl = d["x"], d["uv"], d["bl"]
    n, D = x.shape
    L = uv.shape[0]
    warps, lanes = K["kQueryWarps"], 32
    rows_b = H.transform(x, uv, bl)
    warp_of = (np.arange(n) // lanes) % warps
    got = {("kMaxLshDim", D), ("kMaxTables", L), ("n", n)}
    fills = []
    for key in d["keys"]:
        kh = H.transform(key[None, :], uv, bl)[0]
        cand = np.any(rows_b == kh[None, :], axis=1)
        per_warp = np.bincount(warp_of[cand], minlength=warps)
        fills.append(per_warp)
    fills = np.array(fills)
    if n < warps * lanes:
        assert (np.bincount(warp_of, minlength=warps) == 0).any()      # some warps see no rows
        got.add(("empty_warp", 1))
    for k in d["ks"]:
        got.add(("kMaxK", k))
        if fills.min(axis=1).max() > k:
            got.add(("full_lists", k))
    if d["dup"] is not None:
        assert np.all(fills > max(d["ks"]))                            # every warp's list full, for every key
        assert len(set(warp_of[d["dup"]].tolist())) == warps
        i, dist = H.approx_nearest_neighbors(d["ids"], x, uv, bl, d["keys"][0], 16)
        assert np.all(dist == 0) and len(set(i.tolist())) == 9          # 8 equal ids, 8 distinct: ties at distance 0
        got.add(("cross_warp_ties", 1))
    return got


# ---- ALS --------------------------------------------------------------------------------------------------------
REC_SRC = (1, 31, 32, 33)
REC_DST = (1, 127, 128, 129, 257)
REC_NUM = (1, 31, 32, 33, 127, 128)


def _rec_grid(rank):
    """Random factors with rows equal across the 128-destination tiles (ties go to the lower position)."""
    rng = np.random.default_rng(rank)
    src = rng.standard_normal((max(REC_SRC), rank)).astype(np.float32)
    dst = rng.standard_normal((max(REC_DST), rank)).astype(np.float32)
    for a, b in ((127, 128), (0, 256), (1, 129), (126, 255)):
        dst[b] = dst[a]
    src[30] = 0                                                         # every score 0 for one source
    src[29] = dst[127]                                                  # the planted tie near the top
    ids = (np.arange(max(REC_DST)) * 7 + 2).astype(np.int32)
    return dict(src=src, dst=dst, ids=ids, rank=rank, grid=[(s, t, m) for s in REC_SRC for t in REC_DST
                                                           for m in REC_NUM])


def _rec_reach(d):
    got = {("kMaxRank", d["rank"])}
    for s, t, m in d["grid"]:
        got |= {("kSrcPerBlock", s), ("kTile", t), ("kMaxNum", m)}
    ids, sc = A.recommend(d["src"][:33], d["ids"][:257], d["dst"][:257], 128)
    pos = {int(v): i for i, v in enumerate(ids[29])}
    a, b = pos[int(d["ids"][127])], pos[int(d["ids"][128])]             # equal rows in two tiles, adjacent
    assert b == a + 1 and sc[29, a] == sc[29, b]
    assert ids[30].tolist() == d["ids"][:128].tolist()                 # all ties: positions ascending
    return got


def _rec_overflow():
    """rank 2, entries +-1e20: dots of +inf, -inf and NaN (inf + -inf), finite factors all."""
    big = np.float32(1e20)
    kinds = np.array([[big, big], [-big, -big], [big, -big], [0.5, 0.25]], np.float32)
    pattern = np.random.default_rng(6).integers(0, 4, 300)
    dst = kinds[pattern]
    src = np.array([[big, big], [big, -big], [-big, big], [1.0, 2.0], [0.0, 0.0]], np.float32)
    src = np.r_[src, np.random.default_rng(7).choice([-big, big, 1.0], (28, 2)).astype(np.float32)]
    return dict(src=src, dst=dst, ids=np.arange(300, dtype=np.int32) * 2 + 1, rank=2, nums=[1, 5, 127, 128])


def _overflow_reach(d):
    from oracle import als_cext as X
    ids, sc = X.recommend(d["src"], d["ids"], d["dst"], 128)
    with np.errstate(over="ignore", invalid="ignore"):
        assert np.isposinf(sc).any() and np.isneginf(sc).any() and np.isnan(sc).any()
    mixed = 0
    for row in sc:                                  # NaN ranks as -inf: NaN and -inf interleave, by position
        tail = np.flatnonzero(np.isnan(row) | np.isneginf(row))
        kinds = np.isnan(row[tail])
        mixed += bool(kinds.any() and (~kinds).any() and np.any(kinds[1:] != kinds[:-1]))
    assert mixed >= 2, mixed
    return {("rec_nan", 1), ("rec_inf", 1)}


CHUNK_COUNTS = (1, 31, 32, 33, 64, 65)


def _als_chunks():
    """Users and movies with exactly 1, 31, 32, 33, 64 and 65 ratings; zero ratings at chunk positions 0, 31 and
    32 of a 65-rating user and a 65-rating movie; a movie rated 0 by all its users, so its factor is exactly 0."""
    u, m, r = [], [], []
    rng = np.random.default_rng(31)
    for n, mv in zip(CHUNK_COUNTS, range(2001, 2007)):              # movies by counts: users 1..n
        for usr in range(1, n + 1):
            u.append(usr), m.append(mv), r.append(rng.integers(1, 11) / 2.0)
    for n, usr in zip(CHUNK_COUNTS, range(501, 507)):               # users by counts: movies 1..n
        for mv in range(1, n + 1):
            u.append(usr), m.append(mv), r.append(rng.integers(1, 11) / 2.0)
    u, m, r = np.array(u), np.array(m), np.array(r)
    r[(u == 506) & np.isin(m, [1, 32, 33])] = 0.0                    # user 506's positions 0, 31, 32
    r[(m == 2006) & np.isin(u, [1, 32, 33])] = 0.0                   # movie 2006's positions 0, 31, 32
    zu = np.array([1, 2, 3, 40])
    u, m, r = np.r_[u, zu], np.r_[m, np.full(4, 3000)], np.r_[r, np.zeros(4)]
    return dict(u=u.astype(np.int32), m=m.astype(np.int32), r=r.astype(np.float32), ranks=[1, 33, 64],
                kw=dict(max_iter=2, reg_param=0.05))


def _als_chunks_reach(d):
    from oracle import als_cext as X
    uids, mids, by_movie, by_user = A.layouts(d["u"], d["m"], d["r"])
    got = {("kMaxRank", k) for k in d["ranks"]}
    for side, (off, src, rr) in (("user", by_user), ("movie", by_movie)):
        cnt = np.diff(off)
        assert set(CHUNK_COUNTS) <= set(cnt.tolist()), side
        got |= {("kChunk", c) for c in CHUNK_COUNTS}
        e = int(np.flatnonzero(cnt == 65)[0])
        zeros = np.flatnonzero(rr[off[e]:off[e + 1]] == 0).tolist()
        assert {0, 31, 32} <= set(zeros), (side, zeros)
        got |= {("zero_at", p) for p in (0, 31, 32)}
    fit = X.fit(d["u"], d["m"], d["r"], rank=4, seed=1, **d["kw"])
    zero_rows = np.flatnonzero(np.all(fit[3] == 0, axis=1))
    assert fit[2][zero_rows].tolist() == [3000]                      # a source factor exactly zero
    got.add(("zero_factor", 1))
    return got


def _als_batched():
    d = _als_chunks()
    n = len(d["u"])
    fold = (np.arange(n) * 7 % 3).astype(np.int32)
    ranks = [1, 33, 64]
    models = [dict(rank=ranks[i % 3], max_iter=1 + (i // 3) % 2, reg_param=(0.05, 0.1)[(i // 6) % 2],
                   exclude_fold=(i // 12) % 4 - 1) for i in range(K["kMaxModels"])]
    return dict(d, fold=fold, n_folds=3, models=models)


def _als_batched_reach(d):
    assert len(d["models"]) == K["kMaxModels"]
    assert {m["rank"] for m in d["models"]} == {1, 33, K["kMaxRank"]}
    assert {m["exclude_fold"] for m in d["models"]} == {-1, 0, 1, 2}
    return {("kMaxModels", len(d["models"])), ("kMaxRank", K["kMaxRank"])}


# ---- the sample builder -----------------------------------------------------------------------------------------
GENRE_WORDS = ["G%02d" % i for i in range(24)]


def _fe_movies():
    """24 genre words: movies 1..24 have one genre each, movies 25..40 three."""
    mid = list(range(1, 41))
    genres = [GENRE_WORDS[i] for i in range(24)]
    genres += ["|".join(GENRE_WORDS[(3 * i + j) % 24] for j in range(3)) for i in range(16)]
    return {"movieId": np.array(mid), "title": ["Movie %d (%d)" % (i, 1950 + i) for i in mid], "genres": genres}


FE_TIMESTAMPS = [1, 10, 100, 12, 120, 1000000000, 2, 20, 2000000000, 19, 199, 1999999999, 3, 30, 300000, 29,
                 2147483647, 214748364, 21474836, 9, 99, 999999999, 1234, 12345, 123456, 1234567, 12345678, 123456789]


def _fe_genres():
    rows = []
    # user 1: movies 1..24 in order (one new genre each), then movies again: windows of 12, 13, ..., 24 genres
    for i, mv in enumerate(list(range(1, 25)) + list(range(1, 11))):
        rows.append((1, mv, 4.0, 1000000000 + i))
    # user 2: the genres in another order, with two ratings per new genre
    order = np.random.default_rng(5).permutation(24) + 1
    for i, mv in enumerate(np.repeat(order, 2).tolist()):
        rows.append((2, mv, 4.0 if i % 3 else 2.0, 1100000000 + i))
    # users with 1, 2, 3, 100, 101 and 102 ratings
    rng = np.random.default_rng(8)
    for usr, n in zip(range(10, 16), (1, 2, 3, 100, 101, 102)):
        for i in range(n):
            rows.append((usr, int(rng.integers(1, 41)), int(rng.integers(1, 11)) / 2.0, 1200000000 + int(rng.integers(0, 50))))
    # user 20: timestamps of 1 to 10 digits sharing string prefixes
    for i, t in enumerate(FE_TIMESTAMPS):
        rows.append((20, int(rng.integers(1, 41)), int(rng.integers(5, 11)) / 2.0, t))
    rows = [rows[i] for i in np.random.default_rng(9).permutation(len(rows))]   # file order differs
    u, m, r, t = (np.array(c) for c in zip(*rows))
    ratings = {"userId": u.astype(np.int32), "movieId": m.astype(np.int32), "rating": r.astype(np.float64),
               "timestamp": t.astype(np.int32)}
    return dict(ratings=ratings, movies=_fe_movies())


def window_genre_counts(ratings, movies):
    """Per rating (file order): the number of distinct genres among the positive ratings of its window."""
    year, genres, words = F.movie_table(movies, int(max(ratings["movieId"].max(), movies["movieId"].max())) + 1)
    user, ts = np.asarray(ratings["userId"], np.int64), np.asarray(ratings["timestamp"], np.int64)
    key = I.ts_string_key(ts)
    order = np.lexsort((np.arange(len(user)), key, user))
    out = np.zeros(len(user), np.int64)
    for i, f in enumerate(order):
        lo = i
        while lo > 0 and i - lo < F.WINDOW and user[order[lo - 1]] == user[f]:
            lo -= 1
        seen = set()
        for j in order[lo:i]:
            if ratings["rating"][j] >= 3.5:
                seen |= {g for g in genres[ratings["movieId"][j]].tolist() if g >= 0}
        out[f] = len(seen)
    return out, words


def _fe_genres_reach(d):
    r, mv = d["ratings"], d["movies"]
    nd, words = window_genre_counts(r, mv)
    assert len(words) == K["kMaxGenres"]
    assert {12, 13, K["kMaxGenres"]} <= set(nd.tolist())
    n_per_user = np.bincount(r["userId"])
    assert {1, 2, 3, K["kWindow"], K["kWindow"] + 1, K["kWindow"] + 2} <= set(n_per_user.tolist())
    ts = r["timestamp"][r["userId"] == 20]
    digits = {len(str(t)) for t in ts.tolist()}
    assert digits == set(range(1, 11))
    s = sorted(str(t) for t in ts.tolist())
    assert s != [str(t) for t in sorted(ts.tolist())]                   # string order is not numeric order
    assert any(b.startswith(a) for a, b in zip(s, s[1:]))               # shared prefixes
    # user 1's 13th positive rating opens a window of genres 0..12, one each, inserted in that order: the table
    # was resized at the 13th key, and its top five differ from the 16-slot table's
    b16, b32 = F.genre_buckets([F.java_string_hash(w) for w in GENRE_WORDS[:13]])
    top = lambda nd: np.argsort(F._genre_order_keys(np.arange(13), nd, b16, b32), kind="stable")[:5].tolist()
    assert top(13) != top(12)
    out = {("kMaxGenres", len(words)), ("window_genres", 12), ("window_genres", 13),
           ("window_genres", K["kMaxGenres"]), ("ts_digits", 10)}
    out |= {("kWindow", n) for n in (K["kWindow"], K["kWindow"] + 1, K["kWindow"] + 2)}
    return out


def _fe_top_movie():
    top = K["kMaxMovieSlots"] - 1
    rows = [(1, top, 4.0, 1000000000 + i) for i in range(3)] + [(1, 5, 3.0, 1000000100), (2, top, 2.5, 5),
                                                                 (2, 5, 5.0, 6), (2, top, 4.5, 7)]
    u, m, r, t = (np.array(c) for c in zip(*rows))
    movies = {"movieId": np.array([5, top]), "title": ["Five (1995)", "Top (2001)"], "genres": ["Drama", "Comedy"]}
    return dict(ratings={"userId": u.astype(np.int32), "movieId": m.astype(np.int32), "rating": r.astype(np.float64),
                         "timestamp": t.astype(np.int32)}, movies=movies)


def _fe_top_reach(d):
    top = K["kMaxMovieSlots"] - 1
    assert d["ratings"]["movieId"].max() == top and top in d["movies"]["movieId"].tolist()
    return {("kMaxMovieSlots", top)}


# ---- the FeatureEngineering job and the sample split (featurejob.cu) ---------------------------------------------
# The values the cases are built at.  Literals rather than K: a constant moved without a case at its new value
# fails test_every_bound_has_a_case.
FJ_PROBS, FJ_BUCKETS, FJ_WORDS, FJ_TOKENS = 1 << 16, 10000, 1 << 20, (1 << 29) - 1
FJ_WORDS_PER_ROW, FJ_PARTS, FJ_TOP_MOVIE, FJ_RATINGS = 256, 64, (1 << 24) - 1, 21000000
GRID_BLOCKS = 132 * 64
STRIDE_256, STRIDE_128 = GRID_BLOCKS * 256, GRID_BLOCKS * 128     # elements one grid covers at 256 / 128 threads
SPLITS_THREADS = 1024                                              # fj_splits_kernel's one block
# the tightest (n, eps) of the sweep in test_the_compress_segments_stay_under_their_cap.  2.0 * eps * n is
# 1679.9999999999998 in double, so the host's floor(2 eps n) is 1 679 and its cap 1 689; the walk takes 1 682
# segments, 3 more than that floor (2 more than the exact 1 680).  A cap without its slack of 8 (1 681) fails here.
# At (3e6, 2e-4), where 2 eps n rounds to exactly 1 200, the walk's 1 202 segments fit even that cap.
TIGHT_N, TIGHT_EPS = 3000000, 0.00028


def seg_cap(n, eps):
    """quantiles_of_keys' bound on fj_compress_kernel's segments."""
    return min(n, int(2.0 * eps * n) + 8) + 2


def compress_segments(n, eps):
    """fj_compress_kernel's walk (oracle.feature_job.one_summary_segments), counted: (segments, heads)."""
    e2 = 2.0 * float(eps)
    T = e2 * n

    def delta(j):
        return 0 if j == 0 or j == n - 1 else int(math.floor(e2 * float(j + 1)))

    ns = heads = 0
    j = n - 1
    while True:
        d = delta(j)
        x = T - float(d + 2)
        t = int(math.ceil(x)) if x > 0 else 0
        if 1 <= j <= n - 2 and t <= j - 1:
            a, b = 1, j
            while a < b:
                mid = (a + b) // 2
                if delta(mid) >= d:
                    b = mid
                else:
                    a = mid + 1
            count, stride = (j - max(a, t + 1)) // (t + 1) + 1, t + 1
        else:
            count, stride = 1, min(t, max(j - 1, 0)) + 1
        ns, heads = ns + 1, heads + count
        j -= count * stride
        if j < 1:
            return ns, heads


def query_many(sampled, n, probs, eps):
    """FQ.query_sampled at many probabilities, vectorised over the samples: the first sample but the last with
    maxRank - targetError <= rank <= minRank + targetError, rank = ceil(p n), targetError = ceil(eps n)."""
    v = np.array([s[0] for s in sampled], np.float64)
    g = np.array([s[1] for s in sampled], np.int64)
    d = np.array([s[2] for s in sampled], np.int64)
    minr = np.cumsum(g)[:-1].astype(np.float64)
    maxr = minr + d[:-1]
    target = float(math.ceil(eps * n))
    out = np.empty(len(probs))
    for i, p in enumerate(np.asarray(probs, np.float64).tolist()):
        if p <= eps:
            out[i] = v[0]
        elif p >= 1 - eps:
            out[i] = v[-1]
        else:
            rank = float(math.ceil(p * n))
            ok = (maxr - target <= rank) & (rank <= minr + target)
            out[i] = v[int(np.argmax(ok))] if ok.any() else v[-1]
    return out


def quantiles(values, probs, eps):
    """FQ.one_summary_quantiles, its query vectorised (query_many)."""
    _, sampled, n = FQ.one_summary_samples(values, eps)
    return query_many(sampled, n, probs, eps)


def discretizer_splits(values, num_buckets, eps):
    """FQ.discretizer_splits over `quantiles`."""
    q = quantiles(values, FQ.discretizer_probabilities(num_buckets), eps)
    q[0], q[-1] = -np.inf, np.inf
    _, first = np.unique(q.view(np.uint64), return_index=True)
    s = q[np.sort(first)]
    assert len(s) >= 3 and np.all(s[:-1] < s[1:])
    return s


def _fj_probs():
    """65 536 probabilities on 200 000 values with ties: 0, eps, 1 - eps, 1 and the doubles next to them, p with p n
    an integer, the rest uniform."""
    rng = np.random.default_rng(41)
    n, eps = 200000, 0.01
    x = np.round(rng.standard_normal(n) * 50)                         # about 700 distinct values
    edges = []
    for p in (0.0, eps, 1 - eps, 1.0):
        edges += [p, np.nextafter(p, -1.0), np.nextafter(p, 2.0)]
    edges = [p for p in edges if 0.0 <= p <= 1.0]
    exact = np.arange(1, 2000) * 97 / n                                # p n = 97 k
    rest = rng.random(FJ_PROBS - len(edges) - len(exact))
    return dict(op="quantile", values=x, eps=eps, probs=np.r_[edges, exact, rest])


def _fj_quantile_reach(d):
    n, eps, p = len(d["values"]), d["eps"], d["probs"]
    ns, heads = compress_segments(n, eps)
    cap = seg_cap(n, eps)
    assert ns <= cap
    got = {("kMaxProbs", len(p)), ("segments_margin", cap - ns)}
    if len(p) >= 2 * 128:
        assert {0.0, 1.0, eps, 1 - eps} <= set(p.tolist())
        assert np.any((p * n == np.floor(p * n)) & (p > eps) & (p < 1 - eps))
    if n > STRIDE_256:
        got.add(("keys_stride", 1))
    if heads > STRIDE_256:                                             # fj_expand_kernel runs over the heads
        got.add(("expand_stride", 1))
    if eps == 0.0:
        assert heads == n - 1
        got.add(("every_value_a_head", 1))
    if (n, eps) == (TIGHT_N, TIGHT_EPS):
        assert ns - int(2.0 * eps * n) == 3, ns
        got.add(("tightest_segments", ns))
    return got


def _fj_tight():
    x = np.random.default_rng(42).integers(0, 1 << 40, TIGHT_N).astype(np.float64)
    return dict(op="quantile", values=x, eps=TIGHT_EPS, probs=np.r_[0.0, 0.001, 0.25, 0.5, 0.8, 0.999, 1.0])


def _fj_stride():
    """n = 3 000 000 at eps = 0: every value but the minimum a head, so the keys and the expansion stride."""
    rng = np.random.default_rng(43)
    x = rng.standard_normal(3000000)
    x[:4] = [-0.0, 0.0, np.inf, -np.inf]
    x[4:1000] = 1.5                                                   # a run of equal values
    return dict(op="quantile", values=x, eps=0.0, probs=np.r_[0.0, 1e-7, 1 / 3, 0.5, 0.8, 1 - 1e-7, 1.0])


def _fj_discretizer_passes():
    """Distinct values, so the split count is nq: num_buckets giving nq = 1023, 1024 and 1025, FJ_BUCKETS, and N
    near both ends of the range."""
    x = np.random.default_rng(44).permutation(100000).astype(np.float64) * 0.5
    nq = lambda N: len(FQ.discretizer_probabilities(N))
    want = []
    for target in (SPLITS_THREADS - 1, SPLITS_THREADS, SPLITS_THREADS + 1):
        want.append(next(N for N in range(target - 2, target + 1) if nq(N) == target))
    Ns = want + [2, 3, 4, 5, 11, 9990, 9997, 9998, 9999, FJ_BUCKETS]
    return dict(op="discretizer", values=x, eps=2.5e-5, buckets=Ns)


def _fj_discretizer_duplicates():
    """FJ_BUCKETS buckets over 100 000 values of about 600 distinct (rounded log-normal counts): `distinct` drops
    most of the 10 001 quantiles, well past the first 1024."""
    x = np.round(np.exp(np.random.default_rng(45).standard_normal(100000) * 2.0))
    return dict(op="discretizer", values=x, eps=2.5e-5, buckets=[FJ_BUCKETS, SPLITS_THREADS])


def _fj_discretizer_reach(d):
    got = set()
    for N in d["buckets"]:
        nq = len(FQ.discretizer_probabilities(N))
        s = discretizer_splits(d["values"], N, d["eps"])
        got |= {("kMaxBuckets", N), ("nq", nq)}
        if len(np.unique(d["values"])) == len(d["values"]):
            assert len(s) == nq, (N, nq, len(s))
        else:
            dup = nq - len(s)
            assert dup > SPLITS_THREADS or N < FJ_BUCKETS, dup
            got.add(("dup_past_threads", int(dup > SPLITS_THREADS)))
    return got


def _fj_bucketize():
    """FJ_BUCKETS + 1 splits (-inf, -0.0 and +inf among them); values on every split, on -0.0 and 0.0, at +-inf and
    at the last split; more than one grid of values.  A second, small split set holds 0.0 instead of -0.0."""
    rng = np.random.default_rng(46)
    inner = np.sort(rng.choice(np.arange(-50000, 50000), FJ_BUCKETS - 1, replace=False)).astype(np.float64) / 8
    inner[np.argmin(np.abs(inner))] = -0.0
    splits = np.r_[-np.inf, inner, np.inf]
    assert np.all(splits[:-1] < splits[1:]) and (np.signbit(splits) & (splits == 0)).any()
    n = STRIDE_256 + 300001
    v = rng.uniform(-7000, 7000, n)
    v[:len(splits)] = splits
    v[len(splits):len(splits) + 6] = [-0.0, 0.0, np.inf, -np.inf, -0.0, np.inf]
    rng.shuffle(v)
    small = np.array([-np.inf, -1.0, 0.0, 2.5, np.inf])
    sv = np.array([-0.0, 0.0, -1.0, 2.5, np.inf, -np.inf, 1e300, -1e300, 3.0])
    return dict(op="bucketize", runs=[(splits, v), (small, sv)])


def _fj_bucketize_reach(d):
    (splits, v), _ = d["runs"]
    assert len(splits) == FJ_BUCKETS + 1 and np.isin(splits, v).all() and len(v) > STRIDE_256
    b = FQ.bucketize(splits, v)
    assert b.max() == len(splits) - 2 and b.min() == 0
    return {("n_splits", len(splits)), ("bucket_stride", 1)}


def _fj_scaler():
    """-0.0 and 0.0 the two smallest of more than one grid of values; +-1e308 (a range of +inf: 0 and NaN); a fitted
    min / max with values outside it."""
    rng = np.random.default_rng(47)
    n = STRIDE_256 + 12345
    a = rng.uniform(0, 5, n)
    a[[17, 4000]] = [-0.0, 0.0]
    b = np.r_[1e308, -1e308, 0.0, 5.0, -1e308, 1e308, 1.0]
    return dict(op="scaler", fits=[(a, None), (b, None), (a, (1.0, 3.5)), (b, (2.0, 2.0))])


def _fj_scaler_reach(d):
    a = d["fits"][0][0]
    lo2 = a[np.argsort(FQ._total_order_keys(a), kind="stable")[:2]]
    assert len(a) > STRIDE_256
    with np.errstate(over="ignore", invalid="ignore"):
        s = FQ.min_max_scale(d["fits"][1][0])[0]
    assert np.isnan(s).any() and (s == 0).any()
    return {("scale_stride", 1), ("scale_overflow", 1), ("signed_zero_min", int(np.signbit(lo2).tolist() == [True, False] and not lo2.any()))}


# one movie of FJ_RATINGS - 1 ratings, a at 1 half-star and b at 10, and a one-rating movie at id 0.  Q = 81 a b is
# below 2^53, but n S2 and S1^2 are not: Q formed in double - both products rounded, or either one fused (an FMA) -
# gives another variance at this split
RATING_SPLIT = (10500001, 10499998)


def double_q_forms(N, S1, S2):
    """Q = N S2 - S1^2 with double products: both rounded, and each of the two fused forms."""
    both = float(N) * float(S2) - float(S1) * float(S1)
    return both, float(N * S2 - int(float(S1) * float(S1))), float(int(float(N) * float(S2)) - S1 * S1)


def _fj_ratings():
    a, b = RATING_SPLIT
    movie = np.r_[np.int32(0), np.full(a + b, 7, np.int32)]
    half = np.r_[np.int8(6), np.ones(a, np.int8), np.full(b, 10, np.int8)]
    p = np.random.default_rng(48).permutation(len(movie))
    return dict(op="ratings", movie=movie[p], half=half[p])


def _fj_ratings_reach(d):
    m, h = d["movie"].astype(np.int64), d["half"].astype(np.int64)
    n, s1, s2 = np.bincount(m), np.bincount(m, h).astype(np.int64), np.bincount(m, h * h).astype(np.int64)
    N, S1, S2 = int(n[7]), int(s1[7]), int(s2[7])
    Q = N * S2 - S1 * S1
    assert Q == 81 * RATING_SPLIT[0] * RATING_SPLIT[1] and Q < 2 ** 53
    den = float(4 * N * (N - 1))
    assert all(float(Q) / den != q / den for q in double_q_forms(N, S1, S2))
    assert np.isnan(FQ.rating_features(m, h)[3][0])                    # one rating: a null variance
    return {("kMaxRatings", len(m)), ("rating_q_past_double", 1)}


def _java_hash(s):
    return F.java_string_hash(s)


def trie_keys(hashes):
    """FQ.trie_order_key, vectorised over int32 hashes."""
    h = np.asarray(hashes, np.int64).astype(np.uint32).astype(np.uint64)
    m = np.uint64(0xFFFFFFFF)
    h = (h + (~(h << np.uint64(9)) & m)) & m
    h ^= h >> np.uint64(14)
    h = (h + (h << np.uint64(4))) & m
    h ^= h >> np.uint64(10)
    k = np.zeros_like(h)
    for level in range(7):
        k = (k << np.uint64(5)) | ((h >> np.uint64(5 * level)) & np.uint64(31))
    return k


def _fj_words():
    """FJ_WORDS words: the first 4096 real strings, the rest random hashes with distinct trie keys; counts 1 and 2
    (ties everywhere, so the trie order decides)."""
    rng = np.random.default_rng(49)
    strs = ["w%04d" % i for i in range(4096)]
    h = np.array([_java_hash(s) for s in strs], np.int64)
    extra = rng.integers(-2 ** 31, 2 ** 31, 2 * FJ_WORDS)
    allh = np.r_[h, extra]
    _, first = np.unique(trie_keys(allh), return_index=True)
    keep = np.sort(first)
    assert keep[:4096].tolist() == list(range(4096))
    hashes = allh[keep[:FJ_WORDS]].astype(np.int32)
    counts = rng.integers(1, 3, FJ_WORDS)
    tok = rng.permutation(np.repeat(np.arange(FJ_WORDS, dtype=np.int32), counts))
    return dict(op="indexer", tok=tok, hashes=hashes, strs=strs)


def _fj_count_field():
    """Two words, counts 2^29 - 2 and 1: FJ_TOKENS tokens, the count field full.  The lone word's trie key is the
    smaller, so only the count field puts it second.  The tokens are built by the run (2 GiB)."""
    h = np.array([_java_hash("Drama"), _java_hash("Film-Noir")], np.int32)
    if trie_keys(h)[1] > trie_keys(h)[0]:
        h = h[::-1].copy()
    return dict(op="indexer", counts=[FJ_TOKENS - 1, 1], hashes=h, lone_at=123456789)


def indexer_tokens(d):
    if "tok" in d:
        return d["tok"]
    tok = np.zeros(sum(d["counts"]), np.int32)
    tok[d["lone_at"]] = 1
    return tok


def indexer_oracle(d):
    """The label order, (-count, trie key): FQ.string_indexer_labels' sort, on hashes."""
    cnt = np.bincount(d["tok"], minlength=len(d["hashes"])) if "tok" in d else np.array(d["counts"], np.int64)
    order = np.lexsort((trie_keys(d["hashes"]), -cnt)).astype(np.int32)
    return order, cnt[order].astype(np.int64)


def _fj_indexer_reach(d):
    W, h = len(d["hashes"]), d["hashes"]
    assert len(np.unique(trie_keys(h))) == W
    sub = np.arange(0, 4096 if "strs" in d else W)
    ks = trie_keys(h[sub])
    assert ks.tolist() == [FQ.trie_order_key(int(x)) for x in h[sub].tolist()]
    if "strs" in d:
        assert FQ.hash_trie_keys(d["strs"]) == [d["strs"][i] for i in np.argsort(ks)]
        cnt = np.bincount(d["tok"])
        assert set(cnt.tolist()) == {1, 2}
        return {("kMaxWords", W)}
    assert sum(d["counts"]) == FJ_TOKENS and np.argmin(trie_keys(h)) == 1
    return {("kMaxTokens", sum(d["counts"]))}


def _fj_multi_hot():
    """One movie of FJ_WORDS_PER_ROW genres listed in descending label order (fj_csr_kernel's insertion sort shifts
    every element); 2 171 136 one-genre movies and their words, more than one grid at 256 threads (so fj_hist,
    fj_row_iota, fj_row_len and fj_csr_kernel all stride), ids 0 and FJ_TOP_MOVIE."""
    words = ["g%03d" % i for i in range(FJ_WORDS_PER_ROW)]
    per = 66 * (np.arange(FJ_WORDS_PER_ROW) + 1)                      # word w in 66 (w + 1) one-genre movies
    one = np.repeat(np.arange(FJ_WORDS_PER_ROW), per)
    rng = np.random.default_rng(50)
    n = len(one) + 1
    ids = rng.choice(FJ_TOP_MOVIE - 1, n, replace=False) + 1
    ids[:2] = [0, FJ_TOP_MOVIE]
    genres = ["|".join(words)] + [words[w] for w in one.tolist()]      # the big movie: labels 255, 254, ..., 0
    p = rng.permutation(n)
    return dict(op="multi_hot", ids=ids[p].astype(np.int32), genres=[genres[i] for i in p.tolist()])


def _fj_multi_hot_reach(d):
    lens = np.array([g.count("|") + 1 for g in d["genres"]])
    big = d["genres"][int(np.argmax(lens))].split("|")
    labels, counts = FQ.string_indexer_labels([w for g in d["genres"] for w in g.split("|")])
    index = {w: k for k, w in enumerate(labels)}
    lab = [index[w] for w in big]
    assert lab == sorted(lab, reverse=True) and len(set(counts)) == len(counts)
    assert {0, FJ_TOP_MOVIE} <= set(d["ids"].tolist())
    got = {("kMaxWordsPerRow", int(lens.max())), ("kMaxMovieId", FJ_TOP_MOVIE), ("kMaxMovieId", 0)}
    if len(d["ids"]) > STRIDE_128:
        got.add(("csr_stride", 1))
    if len(d["ids"]) > STRIDE_256:
        got.add(("row_stride", 1))                                    # fj_row_iota_kernel, fj_row_len_kernel
    if lens.sum() > STRIDE_256:
        got.add(("hist_stride", 1))                                   # fj_hist_kernel over the words
    return got


def _fj_split():
    """FJ_PARTS weights from 1e-300 to 1e300, some 0; fraction 0 and 1; n = 1."""
    w = 10.0 ** np.linspace(-300, 300, FJ_PARTS)
    w[[3, 20, 40, 63]] = 0.0
    w[[10, 50]] = [1.0, 1e300]
    return dict(op="split", runs=[(300000, 11, 0.5, w), (300000, 12, 1.0, w), (300000, 13, 0.0, w),
                                  (1, 14, 1.0, w), (200000, 15, 1.0, np.r_[1.0, 0.0, 2.0, 1e-300])])


def _fj_split_reach(d):
    got = {("kMaxParts", max(len(w) for *_, w in d["runs"]))}
    for n, seed, frac, w in d["runs"]:
        parts = FQ.split_samples(n, seed, frac, w)
        assert all(len(p) == 0 for p, x in zip(parts, w) if x == 0)
        got |= {("split_fraction", frac), ("split_n", min(n, 2))}
        if frac == 0:
            assert sum(len(p) for p in parts) == 0
    return got


def _fj_ts_split():
    """Timestamps at +-2^53, negative; all equal (the test part empty); exactly one sampled row."""
    rng = np.random.default_rng(51)
    ts = rng.integers(-10 ** 12, 10 ** 12, 100000)
    ts[:6] = [2 ** 53, -2 ** 53, 2 ** 53, -1, 0, 2 ** 53 - 1]
    ts[6:5000] = 2 ** 53
    u = FQ.stream_uniforms(61, 0, 1000)
    one = float(np.sort(u)[1])                                         # exactly the smallest uniform passes
    return dict(op="ts_split", runs=[(ts, 17, 0.5, 0.01), (ts, 18, 1.0, 0.0), (np.full(5000, -77), 19, 0.3, 0.05),
                                     (np.arange(1000) - 500, 61, one, 0.05)])


def _fj_ts_reach(d):
    got = set()
    for ts, seed, frac, eps in d["runs"]:
        tr, te, split = FQ.split_samples_by_timestamp(ts, seed, frac, eps)
        if len(tr) + len(te) == 1:
            got.add(("ts_one_sampled", 1))
        if len(set(ts.tolist())) == 1:
            assert len(te) == 0
            got.add(("ts_all_equal", 1))
        if np.abs(ts).max() == 2 ** 53:
            assert (ts < 0).any()
            got.add(("ts_2_53", 1))
    return got


# ---- implicit ALS and RankingMetrics (als.cu) --------------------------------------------------------------------
YTY_MEMBERS = (0, 1, 31, 32, 33, 64, 65, 2, 3, 5)                     # entities per YtY block (raw id mod blocks)


def _block_ids(counts, base):
    B = K["kYtyBlocks"]
    assert len(counts) == B, (len(counts), B)
    return np.concatenate([base + b + B * np.arange(c) for b, c in enumerate(counts)]).astype(np.int32)


def _yty_tiles():
    """Users and movies with YTY_MEMBERS entities in the kYtyBlocks YtY blocks; ranks 15 (nA 120, one tile), 16 (136, two)
    and 64 (2080, 17).  Ratings include 0 and negatives."""
    rng = np.random.default_rng(52)
    users, movies = _block_ids(YTY_MEMBERS, 1000), _block_ids(YTY_MEMBERS[::-1], 5000)
    u = np.r_[np.repeat(users, 6), rng.choice(users, len(movies))]
    m = np.r_[rng.choice(movies, 6 * len(users)), movies]
    r = rng.choice([-1.0, 0.0, 0.5, 1.0, 2.5, 4.0, 5.0], len(u)).astype(np.float32)
    return dict(u=u.astype(np.int32), m=m.astype(np.int32), r=r,
                fits=[dict(rank=k, max_iter=2, reg_param=0.05, alpha=a, seed=k) for k, a in ((15, 1.0), (16, 40.0),
                                                                                            (64, 1.0))])


def _yty_reach(d):
    B = K["kYtyBlocks"]
    got = set()
    for ids, want in ((d["u"], YTY_MEMBERS), (d["m"], YTY_MEMBERS[::-1])):
        per = np.bincount(np.unique(ids) % B, minlength=B)
        assert per.tolist() == list(want), per
        got |= {("yty_members", int(c)) for c in per} | {("kYtyBlocks", len(per))}
    for f in d["fits"]:
        nA = f["rank"] * (f["rank"] + 1) // 2
        got.add(("yty_tiles", -(-nA // K["kYtyThreads"])))
    return got


def _implicit_chunks():
    """Users and movies with 31, 32, 33, 64 and 65 ratings; zero and negative ratings at positions 0, 31 and 32 of
    the 33- and 65-rating entities.  At alpha 0 and 40."""
    counts = CHUNK_COUNTS[1:]
    u, m, r = [], [], []
    rng = np.random.default_rng(53)
    for n, mv in zip(counts, range(2001, 2006)):
        for usr in range(1, n + 1):
            u.append(usr), m.append(mv), r.append(rng.integers(1, 11) / 2.0)
    for n, usr in zip(counts, range(501, 506)):
        for mv in range(1, n + 1):
            u.append(usr), m.append(mv), r.append(rng.integers(1, 11) / 2.0)
    u, m, r = np.array(u), np.array(m), np.array(r)
    for usr, vals in ((505, (0.0, -2.0, 0.0)), (503, (-1.0, 0.0, -0.5))):
        for mv, x in zip((1, 32, 33), vals):
            r[(u == usr) & (m == mv)] = x
    for mv, vals in ((2005, (-1.0, 0.0, -3.0)), (2003, (0.0, -4.0, 0.0))):
        for usr, x in zip((1, 32, 33), vals):
            r[(m == mv) & (u == usr)] = x
    fits = [dict(rank=k, max_iter=2, reg_param=0.05, alpha=a, seed=k) for k in (8, 33) for a in (0.0, 40.0)]
    return dict(u=u.astype(np.int32), m=m.astype(np.int32), r=r.astype(np.float32), fits=fits)


def _implicit_chunks_reach(d):
    _, _, by_movie, by_user = A.layouts(d["u"], d["m"], d["r"])
    c = K["kChunk"]
    got = {("implicit_alpha", f["alpha"]) for f in d["fits"]}
    for side, (off, src, rr) in (("user", by_user), ("movie", by_movie)):
        cnt = np.diff(off)
        assert set(CHUNK_COUNTS[1:]) <= set(cnt.tolist()), side
        got |= {("implicit_chunk", int(x)) for x in CHUNK_COUNTS[1:]}
        for e in np.flatnonzero(np.isin(cnt, (c + 1, 2 * c + 1))):
            rs = rr[off[e]:off[e + 1]]
            nonpos = set(np.flatnonzero(rs <= 0).tolist())
            assert {0, c - 1, c} <= nonpos, (side, e, nonpos)
            assert (rs < 0).any() and (rs == 0).any()
            got |= {("implicit_nonpos_at", p) for p in (0, c - 1, c)}
            got |= {("implicit_n_plus", (j // c, int((rs[j:j + c] > 0).sum()))) for j in range(0, len(rs), c)}
    return got


RANK_L = (0, 1, 31, 32, 33, 64, 65)


RANK_HITS = (0, 31, 32, 63, 64)                                      # either side of a 32-wide ballot


def _ranking_lists():
    """Per L in RANK_L, queries whose label sets have 1, 31, 32, 33, L + 3 and 40 distinct ids, one of 100 copies
    of one id, and one empty.  Every set of two or more ids holds the predictions at RANK_HITS (those below L) and
    at L - 1, among misses: its other ids are a few more predictions and ids never predicted.  The one-id sets are
    the prediction at L - 1.  Per L, k in 1, L - 1, L, L + 1 and past every walk."""
    rng = np.random.default_rng(54)
    runs = []
    for L in RANK_L:
        named = sorted({i for i in RANK_HITS if i < L} | ({L - 1} if L else set()))
        labels, preds = [], []
        for q, size in enumerate((1, 31, 32, 33, L + 3, 100, 0, 40)):
            pred = 100000 * (q + 1) + rng.permutation(1000)[:L]
            if size == 0:
                lab = pred[:0]
            elif size in (1, 100):
                lab = np.full(size, pred[L - 1] if L else 7)
            else:
                others = [i for i in rng.permutation(L)[:size // 4].tolist() if i not in named]
                hit = pred[named + others][:size]
                lab = np.r_[hit, 50 + np.arange(size - len(hit))]           # never predicted: misses
                lab = np.r_[lab, lab[:size // 4]]                         # duplicates in the list
            preds.append(pred), labels.append(rng.permutation(lab).astype(np.int32))
        ks = sorted({k for k in (1, L - 1, L, L + 1, 200) if k >= 1})
        runs.append((np.array(preds, np.int32).reshape(len(preds), L), labels, ks, named))
    return dict(runs=runs)


def labels_csr(labels):
    off = np.zeros(len(labels) + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in labels])
    return off, (np.concatenate(labels) if labels else np.zeros(0)).astype(np.int32)


def _ranking_lists_reach(d):
    got = set()
    for pred, labels, ks, named in d["runs"]:
        L = pred.shape[1]
        got.add(("rank_L", L))
        for row, lab in zip(pred.tolist(), labels):
            labset = set(lab.tolist())
            dist = len(labset)
            hits = [i for i, x in enumerate(row) if x in labset]
            if len(lab) == 100 and dist == 1:
                got.add(("rank_repeated_label", 100))
            for k in ks:
                steps = max(L, min(max(L, dist), k)) if dist else 0
                got.add(("rank_steps", steps))
            if dist == 0 or L == 0:
                continue
            if dist == 1:
                assert hits == [L - 1], hits
            else:
                assert set(named) <= set(hits) and (len(hits) < L or L == 1), (L, dist, hits)
                for p in hits:                                        # a hit with a miss before it
                    if p == 0 or len(set(range(p)) - set(hits)):
                        got.add(("rank_hit_at", p))
            for k in ks:                                              # the walks see the hits
                _, ndcg, ap = XP.query_metrics(row, lab, k)
                assert ap > 0 and (ndcg > 0) == (min(hits) < min(max(L, dist), k)), (L, dist, k)
            got.add(("rank_distinct", dist if dist <= 33 else "past_L" if dist > L else dist))
        for k in ks:
            got.add(("rank_k_vs_L", k - L if abs(k - L) <= 1 else "past" if k > 2 * L + 3 else "other"))
    return got


def _ranking_grid():
    """67 585 and 140 000 queries: warps take a second and a third query (grid of 8448 blocks of 8 warps)."""
    rng = np.random.default_rng(55)
    runs = []
    for n in (GRID_BLOCKS * K["kRankWarps"] + 1, 140000):
        pred = rng.integers(0, 40, (n, 10)).astype(np.int32)
        labels = [rng.integers(0, 40, int(c)).astype(np.int32) for c in rng.integers(0, 12, n)]
        runs.append((pred, labels, [10]))
    return dict(runs=runs)


def _ranking_grid_reach(d):
    per_trip = K["kMaxGridBlocks"] * K["kRankWarps"]
    return {("rank_trips", -(-len(p) // per_trip)) for p, _, _ in d["runs"]}


def trips(n, per_trip=STRIDE_256):
    """Grid-stride trips of a 256-thread kernel launched through grid_for over n elements."""
    return -(-int(n) // per_trip)


# ---- BinaryClassificationMetrics (binary_metrics.cu) --------------------------------------------------------------
def segmented_metrics(scores, labels, offsets):
    """BM.BinaryMetrics (numBins 0) of every set at once, vectorised over the sets, for millions of sets.  Returns
    per set n, positives and pt_off [n_sets + 1] (each set's points), per point (the sets' points one after another)
    thresholds, tp, fp, precision, recall and FPR, each set's ROC and PR points (roc_off, pr_off) and their trapezoid
    terms (roc_terms_off, pr_terms_off), and per set both areas (math.fsum of the terms)."""
    s = np.ascontiguousarray(scores, np.float64)
    off = np.asarray(offsets, np.int64)
    S = len(off) - 1
    sizes = np.diff(off)
    sid = np.repeat(np.arange(S), sizes)
    key = BM.descending_key(s)
    order = np.lexsort((key, sid))                               # (set, threshold order), stable
    k, p, g = key[order], BM.is_positive(labels)[order].astype(np.int64), sid[order]
    starts = np.flatnonzero(np.r_[True, (k[1:] != k[:-1]) | (g[1:] != g[:-1])])
    rpos = np.add.reduceat(p, starts)
    rneg = np.diff(np.r_[starts, len(k)]) - rpos
    T = np.bincount(g[starts], minlength=S)
    pt_off = np.r_[0, np.cumsum(T)]
    ctp, cfp = np.cumsum(rpos), np.cumsum(rneg)
    first = pt_off[:-1]
    tp = ctp - np.repeat(ctp[first] - rpos[first], T)
    fp = cfp - np.repeat(cfp[first] - rneg[first], T)
    P = tp[pt_off[1:] - 1]
    Nn = sizes - P
    Pr, Nr = np.repeat(P, T), np.repeat(Nn, T)
    rec = np.where(Pr == 0, 0.0, tp.astype(np.float64) / np.maximum(Pr, 1).astype(np.float64))
    fpr = np.where(Nr == 0, 0.0, fp.astype(np.float64) / np.maximum(Nr, 1).astype(np.float64))
    prec = BM.precision(tp, fp)
    idx = np.arange(S)
    # ROC: (0, 0), (FPR, recall) per point, (1, 1); PR: (0, the first precision), (recall, precision) per point
    roc_off, pr_off = pt_off + 2 * np.arange(S + 1), pt_off + np.arange(S + 1)
    roc = np.empty((roc_off[-1], 2))
    at = np.arange(len(tp)) + 2 * np.repeat(idx, T) + 1
    roc[at] = np.stack([fpr, rec], 1)
    roc[roc_off[:-1]] = 0.0
    roc[roc_off[1:] - 1] = 1.0
    pr = np.empty((pr_off[-1], 2))
    pr[np.arange(len(tp)) + np.repeat(idx, T) + 1] = np.stack([rec, prec], 1)
    pr[pr_off[:-1]] = np.stack([np.zeros(S), prec[first]], 1)

    def terms(pts, poff):
        t = BM.trapezoid_terms(pts)                            # consecutive pairs; drop those across two sets
        keep = np.ones(len(t), bool)
        keep[poff[1:-1] - 1] = False
        return t[keep], poff - np.arange(S + 1)

    roc_t, roc_toff = terms(roc, roc_off)
    pr_t, pr_toff = terms(pr, pr_off)

    def areas(t, toff):
        cnt = np.diff(toff)
        out = np.add.reduceat(t, toff[:-1]) if len(t) else np.zeros(S)
        for i in np.flatnonzero(cnt > 64):                       # long sets: the exactly rounded sum
            out[i] = math.fsum(t[toff[i]:toff[i + 1]])
        return out

    return dict(n=sizes, positives=P, pt_off=pt_off, thresholds=BM.key_score(k[starts]), tp=tp, fp=fp,
                precision=prec, recall=rec, fpr=fpr, roc=roc, roc_off=roc_off, pr=pr, pr_off=pr_off,
                roc_terms=roc_t, roc_terms_off=roc_toff, pr_terms=pr_t, pr_terms_off=pr_toff,
                area_roc=areas(roc_t, roc_toff), area_pr=areas(pr_t, pr_toff))


def set_curves(R, s):
    """Set s's thresholds, tp, fp, ROC, PR, and precision, recall and F1 by threshold, from segmented_metrics."""
    a, b = R["pt_off"][s], R["pt_off"][s + 1]
    thr, prec, rec = R["thresholds"][a:b], R["precision"][a:b], R["recall"][a:b]
    return [thr, R["tp"][a:b], R["fp"][a:b], R["roc"][R["roc_off"][s]:R["roc_off"][s + 1]],
            R["pr"][R["pr_off"][s]:R["pr_off"][s + 1]], np.stack([thr, prec], 1), np.stack([thr, rec], 1),
            np.stack([thr, BM.f_measure(prec, rec, 1.0)], 1)]


def bm_curves(m):
    """The same of BM.BinaryMetrics m."""
    return [m.thresholds(), m.tp, m.fp, m.roc(), m.pr(), m.precision_by_threshold(), m.recall_by_threshold(),
            m.f_measure_by_threshold(1.0)]


def set_bits(n_sets):
    """The set sort's bit count: the width of the largest set index, n_sets - 1."""
    return max(1, int(n_sets - 1).bit_length())


def _bm_run(scores, labels, sizes, path="host", rng=None):
    """One call: the sets of `sizes` pairs.  Full curves are compared on a sample: the first and last sets, the sets
    either side of each power of two, and a few drawn at random."""
    S = len(sizes)
    sample = {0, S - 1} | {v for b in range(1, 32) for v in ((1 << b) - 1, 1 << b) if v < S}
    if rng is not None:
        sample |= set(rng.integers(0, S, 8).tolist())
    return dict(scores=scores, labels=labels, offsets=np.r_[0, np.cumsum(sizes)].astype(np.int64), path=path,
                sample=sorted(sample))


def _bm_two_grids():
    """One set of exactly 2 GRID distinct double scores (STRIDE_256 = GRID), plus 5 000 pairs tied with them."""
    rng = np.random.default_rng(60)
    T = 2 * STRIDE_256
    s = (rng.permutation(T) - T // 3) / 7.0
    s = rng.permutation(np.r_[s, rng.choice(s, 5000)])
    y = rng.choice([0.0, 1.0, 0.5, 0.7], len(s), p=[0.5, 0.4, 0.05, 0.05])
    return dict(runs=[_bm_run(s, y, [len(s)])])


def _bm_sets(counts, seed):
    """Per n_sets in counts, sets of 1 to 3 pairs: scores on five levels with ties, NaN, -0.0 and 0.0."""
    rng = np.random.default_rng(seed)
    runs = []
    for S in counts:
        sizes = rng.integers(1, 4, S)
        n = int(sizes.sum())
        s = rng.integers(0, 5, n) / 4.0
        s[rng.random(n) < 0.02] = np.nan
        s[rng.random(n) < 0.02] = -0.0
        y = rng.integers(0, 2, n).astype(np.float64)
        runs.append(_bm_run(s, y, sizes, rng=rng))
    return dict(runs=runs)


BM_SET_T = (2047, 2048, 2049, 4096, 4097, 65536, 65537)             # thresholds per set: kChunk (2 048) edges, 32 and
                                                                    # 33 chunks


def _bm_chunk_sets():
    """Adjacent sets of BM_SET_T distinct thresholds (and 10 % tied pairs), with sets of 1 to 3 pairs between some."""
    rng = np.random.default_rng(61)
    parts = []
    for T in (3,) + BM_SET_T[:3] + (1,) + BM_SET_T[3:] + (2,):
        v = rng.permutation(T) / T - 0.25
        parts.append(rng.permutation(np.r_[v, rng.choice(v, T // 10)]))
    s = np.concatenate(parts)
    y = (rng.random(len(s)) < 0.3 + 0.4 * (s > 0.3)).astype(np.float64)
    return dict(runs=[_bm_run(s, y, [len(p) for p in parts], rng=rng)])


# float32 bit patterns with an even mantissa: in each pair (b, b + 1) only the last mantissa bit differs
BM_F32_EVEN = (0x00000002, 0x00000010, 0x00800000, 0x3F7FFFFE, 0x3F800000, 0x3DCCCCCC, 0xBF800000, 0xC2C80000,
               0x80000004, 0x7F7FFFFE, 0xFF7FFFFE)


def _bm_f32_adjacent():
    """Device path (float32 scores, int32 labels): each pair of BM_F32_EVEN with the smaller score first in input
    order and the two labels different, beside +-inf, +-0, NaN and random float32 scores; two sets, the second the
    first with its labels flipped."""
    rng = np.random.default_rng(62)
    bits = []
    for b in BM_F32_EVEN:
        lo, hi = (b, b + 1) if b < 0x80000000 else (b + 1, b)       # negative: b + 1 is the smaller
        bits += [lo, hi]
    pairs = np.array(bits, np.uint32).view(np.float32)
    special = np.array([np.inf, -np.inf, 0.0, -0.0, np.nan, 1.0, -1.0], np.float32)
    noise = rng.standard_normal(300).astype(np.float32)
    s = np.r_[pairs, special, noise].astype(np.float32)
    y = np.r_[np.tile([0, 1], len(BM_F32_EVEN)), rng.integers(0, 2, len(special) + len(noise))].astype(np.int32)
    y[1::4] = 2                                                      # any label > 0 is a positive
    return dict(runs=[_bm_run(np.r_[s, s], np.r_[y, 1 - np.minimum(y, 1)], [len(s), len(s)], path="device")],
                n_pairs=len(BM_F32_EVEN))


def _bm_reach(d):
    got = set()
    for run in d["runs"]:
        s, off = run["scores"], run["offsets"]
        S = len(off) - 1
        R = segmented_metrics(s.astype(np.float64), run["labels"].astype(np.float64), off)
        T = np.diff(R["pt_off"])
        got |= {("bm_sets_trips", trips(S)), ("bm_points_trips", trips(len(R["tp"])))}
        if S > 1:
            got.add(("bm_set_bits", set_bits(S)))
            assert (S - 1) >> (set_bits(S) - 1) == 1                    # the top set holds the top bit
        for t in np.unique(T).tolist():
            if t > 1000:
                got |= {("bm_set_thresholds", t), ("bm_set_chunks", -(-t // KB["kChunk"]))}
        if T.max() > STRIDE_256:
            t = int(T.max())
            got |= {("bm_curve_trips", trips(t)), ("bm_curve_trips", trips(t + 1))}
            got.add(("bm_roc_end_trip", (t + 1) // STRIDE_256 + 1))    # ROC's (1, 1) is entry T + 1
        if run["path"] == "device":
            k = BM.descending_key(s.astype(np.float64))
            n = d["n_pairs"]
            lo, hi = s[0:2 * n:2].astype(np.float64), s[1:2 * n:2].astype(np.float64)
            assert np.all(lo < hi)                                       # the smaller first in input order
            x = k[0:2 * n:2] ^ k[1:2 * n:2]
            normal = np.abs(lo) >= np.finfo(np.float32).tiny
            assert np.all(x[normal] == np.uint64(1 << 29)) and normal.sum() >= 6
            got.add(("bm_f32_last_bit", 29))
    return got


def test_segmented_metrics_match_binary_metrics_set_by_set():
    """segmented_metrics against BM.BinaryMetrics on 3 000 small random sets with ties, NaN, +-0 and +-inf, and a
    few long ones: every curve and trapezoid term bit for bit, and the areas."""
    rng = np.random.default_rng(63)
    sizes = np.r_[rng.integers(1, 12, 3000), 700, 3000, 1]
    n = int(sizes.sum())
    special = np.array([np.nan, 0.0, -0.0, np.inf, -np.inf, 0.5, 0.25])
    s = np.where(rng.random(n) < 0.3, special[rng.integers(0, len(special), n)], rng.integers(0, 9, n) / 8.0)
    s[-3000:] = rng.random(3000)
    y = rng.choice([0.0, 1.0, 0.5, 0.7, np.nan, 2.0], n)
    off = np.r_[0, np.cumsum(sizes)]
    R = segmented_metrics(s, y, off)
    for i in range(len(sizes)):
        m = BM.BinaryMetrics(s[off[i]:off[i + 1]], y[off[i]:off[i + 1]])
        assert (R["n"][i], R["positives"][i]) == (m.n, m.positives)
        for a, b in zip(set_curves(R, i), bm_curves(m)):
            assert a.shape == b.shape and np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
        rt = R["roc_terms"][R["roc_terms_off"][i]:R["roc_terms_off"][i + 1]]
        pt = R["pr_terms"][R["pr_terms_off"][i]:R["pr_terms_off"][i + 1]]
        assert np.array_equal(rt, BM.trapezoid_terms(m.roc())) and np.array_equal(pt, BM.trapezoid_terms(m.pr()))
        assert abs(R["area_roc"][i] - m.area_under_roc()) <= 1e-13
        assert abs(R["area_pr"][i] - m.area_under_pr()) <= 1e-13


# ---- the LSH similarity join (lsh.cu) ------------------------------------------------------------------------------
def _join(ids_a, xa, ids_b, xb, uv, bl, threshold):
    return dict(ids_a=np.asarray(ids_a, np.int32), xa=np.asarray(xa, np.float32), ids_b=np.asarray(ids_b, np.int32),
                xb=np.asarray(xb, np.float32), uv=np.asarray(uv, np.float64), bl=float(bl),
                threshold=float(threshold))


def join_buckets(run):
    """Both sides' bucket ids, and per table each A row's run of equal ids among B's (np.searchsorted)."""
    ha, hb = H.transform(run["xa"], run["uv"], run["bl"]), H.transform(run["xb"], run["uv"], run["bl"])
    runs = []
    for j in range(ha.shape[1]):
        sb = np.sort(hb[:, j])
        runs.append(np.searchsorted(sb, ha[:, j], "right") - np.searchsorted(sb, ha[:, j], "left"))
    return ha, hb, runs


def _join_keys_trips():
    """n_b = 70 000, L = 64: n_b L = 4 480 000 (bucket) keys, three grid trips.  A is 500 near-copies of B rows,
    bucket length 1e-4: few collisions beyond a row's own copy."""
    rng = np.random.default_rng(70)
    nb, na, D, L = 70000, 500, 4, 64
    xb = rng.standard_normal((nb, D)).astype(np.float32)
    xa = xb[rng.choice(nb, na, replace=False)] + rng.standard_normal((na, D)).astype(np.float32) * 1e-6
    return dict(runs=[_join(rng.permutation(10 * na)[:na], xa, rng.permutation(2 * nb)[:nb] - nb, xb,
                            H.fit(D, L, seed=70), 1e-4, 0.01)])


def _join_runs_trips():
    """n_a = 2 GRID + 0 rows of D = 1, L = 1: the runs kernel covers n_a + 1 entries in three trips, its sentinel
    len[n_a] alone on the third.  B holds buckets 0 .. 2 999, one row each; all but 3 000 A rows fall in negative
    buckets (empty runs, row 0 and row n_a - 1 among them)."""
    rng = np.random.default_rng(71)
    na, nb = 2 * STRIDE_256, 3000
    xb = (np.arange(nb) + 0.5).astype(np.float32)[:, None]
    xa = -(rng.integers(1, 1 << 20, na) + 0.5)
    hits = rng.choice(np.arange(1, na - 1), 3000, replace=False)
    xa[hits] = rng.integers(0, nb, 3000) + 0.25
    return dict(runs=[_join(rng.permutation(na), xa[:, None], np.arange(nb) * 3, xb, [[1.0]], 1.0, 1.0)])


JOIN_C = (1, 1055, 1056, 1057, 256 * 1056, 256 * 1056 + 1)          # kJoinSegments = 1 056 edges, tiles of 256
JOIN_GROUPS = {1: [(1, 1)], 1055: [(5, 211)], 1056: [(32, 33)], 1057: [(7, 151)], 256 * 1056: [(512, 528)],
               256 * 1056 + 1: [(512, 528), (1, 1)]}                # C = sum of a b over buckets of a A and b B rows


def _join_segments():
    """L = 3, D = 3, unit vectors e0, e1, e2 and bucket length 1: table j's bucket of a row is floor(x[j]).  Per
    run, table 0 and table 2 have C_0 and C_2 candidates, buckets built from JOIN_GROUPS at rows 0, 1, ... on both
    sides, so the groups of the two tables share pairs; table 1 has none (A in bucket -3, B in -4)."""
    rng = np.random.default_rng(72)
    runs = []
    for c0, c2 in ((JOIN_C[0], JOIN_C[1]), (JOIN_C[2], JOIN_C[3]), (JOIN_C[4], JOIN_C[5])):
        na = max(sum(a for a, _ in JOIN_GROUPS[c]) for c in (c0, c2)) + 7
        nb = max(sum(b for _, b in JOIN_GROUPS[c]) for c in (c0, c2)) + 5
        ba, bb = np.full((na, 3), -1.0), np.full((nb, 3), -2.0)
        ba[:, 1], bb[:, 1] = -3.0, -4.0
        for j, c in ((0, c0), (2, c2)):
            ra = rb = 0
            for g, (a, b) in enumerate(JOIN_GROUPS[c]):
                ba[ra:ra + a, j], bb[rb:rb + b, j] = 10 * (g + 1), 10 * (g + 1)
                ra, rb = ra + a, rb + b
        xa = ba + 0.5 + (rng.random(ba.shape) - 0.5) * 0.4
        xb = bb + 0.5 + (rng.random(bb.shape) - 0.5) * 0.4
        runs.append(_join(rng.permutation(3 * na)[:na], xa, rng.permutation(3 * nb)[:nb], xb, np.eye(3), 1.0, 1e9))
    return dict(runs=runs)


def _join_extreme_ids():
    """Ids INT32_MIN, -1, 0 and INT32_MAX on both sides, every pair in one bucket: the output order at the sign bit."""
    rng = np.random.default_rng(73)
    ext = np.array([-2 ** 31, -1, 0, 2 ** 31 - 1], np.int64)
    mid = rng.choice(np.r_[np.arange(-2 ** 31 + 1, -2 ** 31 + 50), np.arange(1, 100), 2 ** 31 - 50 + np.arange(49)],
                     60, replace=False)
    ids_a, ids_b = rng.permutation(np.r_[ext, mid[:30]]), rng.permutation(np.r_[ext, mid[30:]])
    xa, xb = rng.random((34, 2)), rng.random((34, 2))                    # nonnegative: every bucket id 0
    return dict(runs=[_join(ids_a, xa, ids_b, xb, _nonneg_unit(2, 2, 73), 1e6, 1e9)])


def _join_signed_zero():
    """Bucket length 1e300 and coordinates +-1e-38, +-1 and 0 on unit vectors e0, e1 and (0.6, 0.8): quotients that
    underflow to -0.0 and +0.0 (floor keeps the sign), and -1.  A -0.0 and a +0.0 are one bucket in every table."""
    rng = np.random.default_rng(74)
    vals = np.array([1e-38, -1e-38, 1.0, -1.0, 0.0], np.float32)
    uv = np.array([[1.0, 0.0], [0.0, 1.0], [0.6, 0.8]])
    return dict(runs=[_join(np.arange(300) * 2 - 299, rng.choice(vals, (300, 2)), np.arange(280) * 5 - 700,
                            rng.choice(vals, (280, 2)), uv, 1e300, 10.0)])


def _join_infinite():
    """Bucket length 5e-324 (the smallest subnormal): coordinates +-1 give buckets +-inf, 0 gives 0 and 1e-30 a
    finite one near 2e293."""
    rng = np.random.default_rng(75)
    vals = np.array([1.0, -1.0, 0.0, 1e-30, -1e-30], np.float32)
    uv = np.array([[1.0, 0.0], [0.0, 1.0], [0.6, 0.8]])
    return dict(runs=[_join(rng.permutation(1000)[:250], rng.choice(vals, (250, 2)), rng.permutation(1000)[:260],
                            rng.choice(vals, (260, 2)), uv, 5e-324, 10.0)])


def _join_reach(d):
    got = set()
    for run in d["runs"]:
        ha, hb, runs = join_buckets(run)
        na, nb, L = len(ha), len(hb), ha.shape[1]
        C = [int(r.sum()) for r in runs]
        assert sum(C) > 0
        got |= {("join_hash_trips", trips(max(na, nb) * L)), ("join_keys_trips", trips(nb * L)),
                ("join_runs_trips", trips(na + 1))}
        if trips(na + 1) > 1:
            got.add(("join_sentinel_trip", na // STRIDE_256 + 1))         # len[n_a] at r = n_a
            assert runs[0][0] == 0 and runs[0][-1] == 0 and 1000 <= (runs[0] > 0).sum() <= 10000
            got |= {("join_empty_run_at", "first"), ("join_empty_run_at", "last")}
        if L == 3 and run["bl"] == 1.0:                                  # the segment runs
            got |= {("join_C", c) for c in C}
            assert C[1] == 0 and C[0] > 0 and C[2] > 0
            got.add(("join_empty_table_between", 1))
            both = (ha[:, None, 0] == hb[None, :, 0]) & (ha[:, None, 2] == hb[None, :, 2])
            assert both.any()                                            # pairs the first-table rule removes
            got.add(("join_first_table_removes", 1))
        ids = set(run["ids_a"].tolist()) & set(run["ids_b"].tolist())
        for v in (-2 ** 31, -1, 0, 2 ** 31 - 1):
            if v in ids and run["bl"] == 1e6:
                assert np.all(ha == ha[0, 0]) and np.all(hb == ha[0, 0])  # one bucket: every pair
                got.add(("join_id", v))
        zero_a, zero_b = ha == 0, hb == 0
        if (zero_a & np.signbit(ha)).any() and (zero_b & ~np.signbit(hb)).any():
            assert (zero_b & np.signbit(hb)).any() and (zero_a & ~np.signbit(ha)).any()
            # a pair whose table-0 ids are -0.0 and +0.0 and that meets again in a later table
            a0 = np.flatnonzero(zero_a[:, 0] & np.signbit(ha[:, 0]))
            b0 = np.flatnonzero(zero_b[:, 0] & ~np.signbit(hb[:, 0]))
            assert np.any(ha[a0][:, None, 1:] == hb[b0][None, :, 1:])
            got.add(("join_signed_zero", 1))
        for inf in (np.inf, -np.inf):
            if (ha == inf).any():
                assert any(((ha[:, j] == inf).sum() * (hb[:, j] == inf).sum()) > 0 for j in range(L))
                got.add(("join_infinite_bucket", inf))
    return got


# ---- nonnegative ALS (als.cu's NNLS tail) --------------------------------------------------------------------------
# rank -> (users, seed): 1 500 ratings of 200 movies drawn with the seed (as nnls_cases()["ill_conditioned"]), the
# init at the same seed, regParam 1e-9: the first movie half-step has a movie that stops at iterMax = max(400, 20 k)
NNLS_ITER_MAX = {19: (20, 6), 20: (40, 4), 21: (30, 8)}
NNLS_REG = 1e-9
# the rank-21 system of the batched fit, whose seed is 6: ratings drawn with seed 1, ids from 1 000
NNLS_BATCH_21 = (30, 1, 1000)


def nnls_ratings(users, seed, first_id=0):
    rng = np.random.default_rng(seed)
    u, m, r = rng.integers(0, users, 1500), rng.integers(0, 200, 1500), rng.integers(1, 11, 1500) / 2.0
    return (u + first_id).astype(np.int32), (m + first_id).astype(np.int32), r.astype(np.float32)


def nnls_first_half(u, m, r, k, seed):
    """The first movie half-step (C oracle) with each movie's NNLS iterations, and its system (Am, B)."""
    from oracle import als_cext as X
    from oracle import als_nnls_cext as XN
    uids, mids, by_movie, _ = A.layouts(u, m, r)
    U = X.init_user_factors(uids, k, seed)
    it = np.zeros(len(mids), np.int32)
    out, _ = XN.solve_half(by_movie, U, uids, k, NNLS_REG, None, it)
    Am, B = A.normal_equations(by_movie, U, k, NNLS_REG)
    return out, it, np.triu(Am) + np.transpose(np.triu(Am, 1), (0, 2, 1)), B


def movies_changed_by(Am, B, rule):
    """The movies whose float32 factor changes when N.nnls runs under `rule` for iterMax instead of max(400, 20k)."""
    x0, _ = N.nnls(Am, B)
    keep = N.iter_max
    N.iter_max = rule
    try:
        x1, _ = N.nnls(Am, B)
    finally:
        N.iter_max = keep
    return int(np.any(x0.astype(np.float32) != x1.astype(np.float32), axis=1).sum())


NNLS_RULES = {"20k": lambda k: 20 * k, "400": lambda k: 400}


def iter_max_reach(u, m, r, k, seed, rules, exactly_one):
    out, it, Am, B = nnls_first_half(u, m, r, k, seed)
    assert (it == N.iter_max(k)).any() and (it < N.iter_max(k)).any(), (k, it.max())
    x, its = N.nnls(Am, B)
    assert np.array_equal(its, it) and np.array_equal(x.astype(np.float32).view(np.uint32), out.view(np.uint32))
    got = {("nnls_iter_max", k)}
    for name in rules:
        assert NNLS_RULES[name](k) < N.iter_max(k)
        changed = movies_changed_by(Am, B, NNLS_RULES[name])
        assert changed == 1 if exactly_one else changed >= 1, (k, name, changed)
        got.add(("nnls_iter_max_rule", name))
    return got


def _nnls_iter_max(k):
    u, m, r = nnls_ratings(*NNLS_ITER_MAX[k])
    return dict(u=u, m=m, r=r, fits=[dict(rank=k, max_iter=1, reg_param=NNLS_REG, seed=NNLS_ITER_MAX[k][1])])


def _nnls_iter_max_reach(d):
    k = d["fits"][0]["rank"]
    rules = {19: ["20k"], 20: [], 21: ["400"]}[k]
    return iter_max_reach(d["u"], d["m"], d["r"], k, d["fits"][0]["seed"], rules, True)


NNLS_BATCH_RANKS = (1, 19, 21, 33, 64)


def _nnls_batch(chol):
    """kMaxModels models over three blocks of disjoint ids: the rank-19 iterMax system (fold 0), NNLS_BATCH_21 (fold
    1) and 600 ratings in folds 0..2, where user 5000 rates only in fold 2 and movie 5000 is rated only in fold 1.
    Ranks NNLS_BATCH_RANKS, max_iter 1 and 2, every excluded fold; models 0 and 1 are the iterMax systems (rank 19
    without fold 1, rank 21 without fold 0).  `chol` holds the models fitted by Cholesky rather than NNLS."""
    rng = np.random.default_rng(76)
    u19, m19, r19 = nnls_ratings(*NNLS_ITER_MAX[19])
    u21, m21, r21 = nnls_ratings(*NNLS_BATCH_21)
    ue = np.r_[rng.integers(5001, 5040, 600), np.full(5, 5000), rng.integers(5001, 5040, 4)]
    me = np.r_[rng.integers(5001, 5060, 600), rng.integers(5001, 5060, 5), np.full(4, 5000)]
    re = rng.integers(0, 11, len(ue)) / 2.0
    fe = np.r_[rng.integers(0, 3, 600), np.full(5, 2), np.full(4, 1)]
    u, m = np.r_[u19, u21, ue].astype(np.int32), np.r_[m19, m21, me].astype(np.int32)
    r = np.r_[r19, r21, re].astype(np.float32)
    fold = np.r_[np.zeros(1500), np.ones(1500), fe].astype(np.int32)
    models = [dict(rank=NNLS_BATCH_RANKS[i % 5], max_iter=1 + (i // 5) % 2, reg_param=(0.05, 0.01)[(i // 40) % 2],
                   exclude_fold=(i // 10) % 4 - 1) for i in range(K["kMaxModels"])]
    models[0] = dict(rank=19, max_iter=1, reg_param=NNLS_REG, exclude_fold=1)
    models[1] = dict(rank=21, max_iter=1, reg_param=NNLS_REG, exclude_fold=0)
    for i, spec in enumerate(models):
        spec["nonnegative"] = i not in chol
        if i in chol and spec["reg_param"] == NNLS_REG:
            spec["reg_param"] = 0.05
    return dict(u=u, m=m, r=r, fold=fold, n_folds=3, models=models, seed=NNLS_ITER_MAX[19][1])


def _nnls_batch_reach(d):
    ms = d["models"]
    assert len(ms) == K["kMaxModels"] and {s["rank"] for s in ms} == set(NNLS_BATCH_RANKS)
    assert {s["max_iter"] for s in ms} == {1, 2} and {s["exclude_fold"] for s in ms} == {-1, 0, 1, 2}
    nn = sum(s["nonnegative"] for s in ms)
    got = {("kMaxModels", len(ms)), ("nnls_batch_mix", (len(ms) - nn, nn))}
    for s in ms:                                                     # an entity with no training rating
        rows = d["fold"] != s["exclude_fold"]
        if s["nonnegative"] and (len(np.unique(d["u"][rows])) < len(np.unique(d["u"]))
                                 or len(np.unique(d["m"][rows])) < len(np.unique(d["m"]))):
            got.add(("nnls_batch_untrained_entity", 1))
    for i, k, (users, seed, first) in ((0, 19, NNLS_ITER_MAX[19] + (0,)), (1, 21, NNLS_BATCH_21)):
        if ms[i]["nonnegative"] and ms[i]["reg_param"] == NNLS_REG:
            assert ms[i]["rank"] == k and ms[i]["max_iter"] == 1
            u, m, r = nnls_ratings(users, seed, first)
            reach = iter_max_reach(u, m, r, k, d["seed"], {19: ["20k"], 21: ["400"]}[k], False)
            got |= {("batch_" + a, b) for a, b in reach}
    return got


def _nnls_singular():
    """singular_case() at regParam 0 in a batch of an NNLS model and a Cholesky model on the same rows, in both
    orders: user 9's system is all zero, singular for Cholesky and not for NNLS."""
    from test_als_oracle import singular_case
    u, m, r = singular_case()
    fold = (np.arange(len(u)) % 2).astype(np.int32)
    spec = dict(rank=2, max_iter=1, reg_param=0.0, exclude_fold=-1)
    return dict(u=u.astype(np.int32), m=m.astype(np.int32), r=r.astype(np.float32), fold=fold, n_folds=2, seed=0,
                orders=[[dict(spec, nonnegative=True), dict(spec, nonnegative=False)],
                        [dict(spec, nonnegative=False), dict(spec, nonnegative=True)]])


def nnls_singular_oracle(d):
    """Per order, the batched fit's message: the Cholesky model's index in the caller's order and its singular
    entity, as the C oracle's single fit reports it; the NNLS single fit has no singular system."""
    from oracle import als_cext as X
    from oracle import als_nnls_cext as XN
    out = []
    for models in d["orders"]:
        for i, s in enumerate(models):
            kw = dict(rank=s["rank"], max_iter=s["max_iter"], reg_param=s["reg_param"], seed=d["seed"])
            if s["nonnegative"]:
                XN.fit(d["u"], d["m"], d["r"], **kw)
                continue
            with pytest.raises(A.SingularError) as e:
                X.fit(d["u"], d["m"], d["r"], **kw)
            out.append("model %d: singular normal equations for %s %d in iteration %d"
                       % (i, e.value.side, e.value.entity_id, e.value.iteration))
    return out


def _nnls_singular_reach(d):
    want = nnls_singular_oracle(d)
    assert [w.split(":")[0] for w in want] == ["model 1", "model 0"]
    return {("nnls_singular_after_nnls", 1)}


# ---- the table --------------------------------------------------------------------------------------------------
BOUNDS = {
    "i2v_depth24_d64_w5_p1": Case("item2vec", lambda: _caterpillar(24, 64, 5, 1, 7), _i2v_reach),
    "i2v_depth24_d33_w1_p64": Case("item2vec", lambda: _caterpillar(24, 33, 1, 64, 8), _i2v_reach),
    "i2v_depth26_d1_w1_p1": Case("item2vec", lambda: _caterpillar(26, 1, 1, 1, 9), _i2v_reach),
    "i2v_depth%d_d1_w1_p64" % DEEPEST: Case("item2vec", lambda: _caterpillar(DEEPEST, 1, 1, 64, 10), _i2v_reach),
    "i2v_sentences_1000_1001_long_window": Case("item2vec", _sentence_edges, _i2v_reach),
    "graph_walks_depth24": Case("graph", _hub_depth_graph, _graph_reach),
    "graph_top_ids_hub_row": Case("graph", _top_id_hub_graph, _graph_reach),
    "lsh_full_lists_cross_warp_ties": Case("lsh", _lsh_full, _lsh_reach),
    "lsh_fewer_rows_than_threads": Case("lsh", _lsh_small, _lsh_reach),
    "lsh_d65_l9": Case("lsh", lambda: _lsh_wide(65, 9, 5000, 1.5), _lsh_reach),
    "lsh_d1024_l64": Case("lsh", lambda: _lsh_wide(1024, 64, 3000, 12.0), _lsh_reach),
    "als_recommend_tiles_rank1": Case("als", lambda: _rec_grid(1), _rec_reach),
    "als_recommend_tiles_rank64": Case("als", lambda: _rec_grid(64), _rec_reach),
    "als_recommend_overflow": Case("als", _rec_overflow, _overflow_reach),
    "als_fit_chunk_edges": Case("als", _als_chunks, _als_chunks_reach),
    "als_fit_64_models": Case("als", _als_batched, _als_batched_reach),
    "featureeng_24_genres_windows_timestamps": Case("featureeng", _fe_genres, _fe_genres_reach),
    "featureeng_top_movie_id": Case("featureeng", _fe_top_movie, _fe_top_reach),
    "fj_quantile_65536_probabilities": Case("featurejob", _fj_probs, _fj_quantile_reach),
    "fj_quantile_tightest_segment_cap": Case("featurejob", _fj_tight, _fj_quantile_reach),
    "fj_quantile_grid_stride_eps0": Case("featurejob", _fj_stride, _fj_quantile_reach),
    "fj_discretizer_splits_kernel_passes": Case("featurejob", _fj_discretizer_passes, _fj_discretizer_reach),
    "fj_discretizer_duplicates_past_1024": Case("featurejob", _fj_discretizer_duplicates, _fj_discretizer_reach),
    "fj_bucketize_10001_splits_grid_stride": Case("featurejob", _fj_bucketize, _fj_bucketize_reach),
    "fj_scaler_signed_zeros_overflow_stride": Case("featurejob", _fj_scaler, _fj_scaler_reach),
    "fj_rating_features_max_ratings": Case("featurejob", _fj_ratings, _fj_ratings_reach),
    "fj_string_indexer_max_words": Case("featurejob", _fj_words, _fj_indexer_reach),
    "fj_string_indexer_count_field": Case("featurejob", _fj_count_field, _fj_indexer_reach),
    "fj_multi_hot_256_words_top_ids_stride": Case("featurejob", _fj_multi_hot, _fj_multi_hot_reach),
    "fj_split_64_parts": Case("featurejob", _fj_split, _fj_split_reach),
    "fj_split_by_timestamp_edges": Case("featurejob", _fj_ts_split, _fj_ts_reach),
    "als_implicit_yty_tiles": Case("als_implicit", _yty_tiles, _yty_reach),
    "als_implicit_solve_chunks": Case("als_implicit", _implicit_chunks, _implicit_chunks_reach),
    "ranking_lists_ballot_passes": Case("ranking_metrics", _ranking_lists, _ranking_lists_reach),
    "ranking_grid_trips": Case("ranking_metrics", _ranking_grid, _ranking_grid_reach),
    "bm_two_grids_of_thresholds": Case("binary_metrics", _bm_two_grids, _bm_reach),
    "bm_4194304_sets": Case("binary_metrics", lambda: _bm_sets([1 << 22], 64), _bm_reach),
    "bm_4194305_sets": Case("binary_metrics", lambda: _bm_sets([(1 << 22) + 1], 65), _bm_reach),
    "bm_2_3_65536_65537_sets": Case("binary_metrics", lambda: _bm_sets([2, 3, 1 << 16, (1 << 16) + 1], 66),
                                    _bm_reach),
    "bm_sets_at_chunk_edges": Case("binary_metrics", _bm_chunk_sets, _bm_reach),
    "bm_float32_last_mantissa_bit": Case("binary_metrics", _bm_f32_adjacent, _bm_reach),
    "lsh_join_keys_three_trips": Case("lsh_join", _join_keys_trips, _join_reach),
    "lsh_join_runs_three_trips": Case("lsh_join", _join_runs_trips, _join_reach),
    "lsh_join_segment_edges": Case("lsh_join", _join_segments, _join_reach),
    "lsh_join_int32_extreme_ids": Case("lsh_join", _join_extreme_ids, _join_reach),
    "lsh_join_signed_zero_buckets": Case("lsh_join", _join_signed_zero, _join_reach),
    "lsh_join_infinite_buckets": Case("lsh_join", _join_infinite, _join_reach),
    "als_nonnegative_iter_max_rank19": Case("als_nonnegative", lambda: _nnls_iter_max(19), _nnls_iter_max_reach),
    "als_nonnegative_iter_max_rank20": Case("als_nonnegative", lambda: _nnls_iter_max(20), _nnls_iter_max_reach),
    "als_nonnegative_iter_max_rank21": Case("als_nonnegative", lambda: _nnls_iter_max(21), _nnls_iter_max_reach),
    "als_nonnegative_batch_64_nnls": Case("als_nonnegative", lambda: _nnls_batch(set()), _nnls_batch_reach),
    "als_nonnegative_batch_1_cholesky_63_nnls": Case("als_nonnegative", lambda: _nnls_batch({37}),
                                                     _nnls_batch_reach),
    "als_nonnegative_batch_63_cholesky_1_nnls": Case("als_nonnegative",
                                                     lambda: _nnls_batch(set(range(K["kMaxModels"])) - {1}),
                                                     _nnls_batch_reach),
    "als_nonnegative_singular_after_nnls": Case("als_nonnegative", _nnls_singular, _nnls_singular_reach),
}


@functools.lru_cache(maxsize=None)
def data(name):
    return BOUNDS[name].make()


@functools.lru_cache(maxsize=None)
def reached(name):
    return frozenset(BOUNDS[name].reach(data(name)))


@pytest.mark.parametrize("name", sorted(BOUNDS))
def test_case_reaches_its_edge(name):
    assert reached(name)


def test_every_bound_has_a_case():
    have = set().union(*(reached(n) for n in BOUNDS))
    need = set()
    need |= {("kMaxRank", 1), ("kMaxRank", K["kMaxRank"]), ("kMaxNum", 1), ("kMaxNum", K["kMaxNum"])}
    need |= {("kTile", t) for t in (1, K["kTile"] - 1, K["kTile"], K["kTile"] + 1, 2 * K["kTile"] + 1)}
    need |= {("kSrcPerBlock", s) for s in (1, K["kSrcPerBlock"] - 1, K["kSrcPerBlock"], K["kSrcPerBlock"] + 1)}
    need |= {("kMaxNum", m) for m in (K["kSrcPerBlock"] - 1, K["kSrcPerBlock"], K["kSrcPerBlock"] + 1,
                                      K["kMaxNum"] - 1)}                 # 32 list entries per lane pass
    c = K["kChunk"]
    need |= {("kChunk", v) for v in (1, c - 1, c, c + 1, 2 * c, 2 * c + 1)}
    need |= {("zero_at", p) for p in (0, c - 1, c)} | {("zero_factor", 1)}
    need |= {("kMaxModels", K["kMaxModels"])}
    need |= {("kMaxK", v) for v in (1, K["kMaxK"] - 1, K["kMaxK"])} | {("full_lists", K["kMaxK"])}
    need |= {("kMaxLshDim", K["kMaxLshDim"]), ("kMaxLshDim", 65), ("kMaxTables", K["kMaxTables"]),
             ("kMaxTables", 9), ("empty_warp", 1), ("cross_warp_ties", 1)}
    need |= {("kMaxCode", d) for d in (24, DEEPEST)} | {("kMaxDim", v) for v in (1, 33, K["kMaxDim"])}
    need |= {("partitions", 1), ("partitions", 64), ("sentence", 1000), ("sentence", 1001), ("window>sentence", 1)}
    need |= {("kMaxGenres", K["kMaxGenres"]), ("window_genres", 12), ("window_genres", 13),
             ("window_genres", K["kMaxGenres"]), ("ts_digits", 10)}
    need |= {("kWindow", K["kWindow"] + i) for i in range(3)} | {("kMaxMovieSlots", K["kMaxMovieSlots"] - 1)}
    need |= {("kIdMask", K["kIdMask"]), ("kIdMask", K["kIdMask"] - 1), ("walk_length", 1), ("rec_nan", 1)}
    assert ("walk_depth", 24) in have or any(k == "walk_depth" and v >= 24 for k, v in have)
    assert any(k == "hub_row" and v >= 5000 for k, v in have)
    # featurejob.cu
    need |= {("kMaxProbs", K["kMaxProbs"]), ("kMaxBuckets", K["kMaxBuckets"]), ("nq", K["kMaxBuckets"] + 1)}
    need |= {("kMaxBuckets", b) for b in (2, K["kMaxBuckets"] - 1)} | {("n_splits", K["kMaxBuckets"] + 1)}
    need |= {("nq", q) for q in (SPLITS_THREADS - 1, SPLITS_THREADS, SPLITS_THREADS + 1)} | {("dup_past_threads", 1)}
    need |= {("kMaxWords", K["kMaxWords"]), ("kMaxTokens", K["kMaxTokens"]), ("kMaxParts", K["kMaxParts"])}
    need |= {("kMaxWordsPerRow", K["kMaxWordsPerRow"]), ("kMaxMovieId", K["kMaxMovieId"]), ("kMaxMovieId", 0)}
    need |= {("kMaxRatings", K["kMaxRatings"]), ("rating_q_past_double", 1)}
    need |= {("tightest_segments", compress_segments(TIGHT_N, TIGHT_EPS)[0]), ("every_value_a_head", 1)}
    need |= {("segments_margin", seg_cap(TIGHT_N, TIGHT_EPS) - compress_segments(TIGHT_N, TIGHT_EPS)[0])}
    assert GRID_BLOCKS == K["kMaxGridBlocks"]
    need |= {("keys_stride", 1), ("expand_stride", 1), ("bucket_stride", 1), ("scale_stride", 1), ("csr_stride", 1),
             ("row_stride", 1), ("hist_stride", 1)}
    need |= {("scale_overflow", 1), ("signed_zero_min", 1)}
    need |= {("split_fraction", f) for f in (0.0, 1.0)} | {("split_n", 1)}
    need |= {("ts_one_sampled", 1), ("ts_all_equal", 1), ("ts_2_53", 1)}
    # implicit ALS and RankingMetrics (als.cu)
    t = K["kYtyThreads"]
    need |= {("yty_tiles", v) for v in (1, 2, -(-(64 * 65 // 2) // t))}
    need |= {("yty_members", v) for v in (0, 1, c - 1, c, c + 1, 2 * c, 2 * c + 1)} | {("kYtyBlocks", K["kYtyBlocks"])}
    need |= {("implicit_chunk", v) for v in (c - 1, c, c + 1, 2 * c, 2 * c + 1)}
    need |= {("implicit_nonpos_at", p) for p in (0, c - 1, c)}
    need |= {("implicit_alpha", 0.0), ("implicit_alpha", 40.0)}
    need |= {("rank_L", v) for v in (0, 1, 31, 32, 33, 64, 65)} | {("rank_repeated_label", 100)}
    need |= {("rank_distinct", v) for v in (1, 31, 32, 33, "past_L")}
    need |= {("rank_k_vs_L", v) for v in (-1, 0, 1, "past")} | {("rank_steps", v) for v in (31, 32, 33, 64, 65)}
    need |= {("rank_hit_at", p) for p in RANK_HITS} | {("rank_trips", 2), ("rank_trips", 3)}
    # binary_metrics.cu: grid trips, the set sort's bits, the area chunks and the float32 sort's first bit
    assert STRIDE_256 == KB["kMaxGridBlocks"] * KB["kChunkThreads"]
    cb = KB["kChunk"]
    need |= {("bm_points_trips", 2), ("bm_curve_trips", 2), ("bm_curve_trips", 3), ("bm_roc_end_trip", 3),
             ("bm_sets_trips", 2)}
    need |= {("bm_set_bits", b) for b in (1, 2, 16, 17, 22, 23)}
    need |= {("bm_set_thresholds", t) for t in (cb - 1, cb, cb + 1, 2 * cb, 2 * cb + 1, 32 * cb, 32 * cb + 1)}
    need |= {("bm_set_chunks", c) for c in (1, 2, 3, 32, 33)} | {("bm_f32_last_bit", 29)}
    # lsh.cu's join: grid trips, the segment walk, the sentinel, empty runs and tables, ids and bucket ids
    G, TJ = K["kJoinSegments"], K["kJoinThreads"]
    need |= {("join_C", c) for c in (1, G - 1, G, G + 1, TJ * G, TJ * G + 1)}
    need |= {("join_keys_trips", 3), ("join_hash_trips", 3), ("join_runs_trips", 3), ("join_sentinel_trip", 3)}
    need |= {("join_empty_run_at", "first"), ("join_empty_run_at", "last"), ("join_empty_table_between", 1),
             ("join_first_table_removes", 1), ("join_signed_zero", 1)}
    need |= {("join_id", v) for v in (-2 ** 31, -1, 0, 2 ** 31 - 1)}
    need |= {("join_infinite_bucket", np.inf), ("join_infinite_bucket", -np.inf)}
    # als.cu's NNLS: iterMax either side of max(400, 20 k), and the batched fit's NNLS slice
    need |= {("nnls_iter_max", k) for k in (19, 20, 21)} | {("nnls_iter_max_rule", r) for r in ("20k", "400")}
    need |= {("batch_nnls_iter_max", 19), ("batch_nnls_iter_max", 21), ("nnls_batch_untrained_entity", 1)}
    need |= {("nnls_batch_mix", (0, K["kMaxModels"])), ("nnls_batch_mix", (1, K["kMaxModels"] - 1)),
             ("nnls_batch_mix", (K["kMaxModels"] - 1, 1)), ("nnls_singular_after_nnls", 1)}
    assert need <= have, sorted(need - have)
    # the deepest case is the deepest code the rating bound allows: one level more needs more ratings than it takes
    assert sum(_deepest_counts(DEEPEST + 1)) > MAX_RATINGS >= sum(_deepest_counts(DEEPEST))
    assert DEEPEST < K["kMaxCode"]


def test_the_constants_are_parsed():
    for name in ("kMaxRank", "kMaxNum", "kTile", "kChunk", "kSrcPerBlock", "kMaxModels", "kMaxK", "kMaxLshDim",
                 "kMaxTables", "kQueryWarps", "kMaxCode", "kMaxDim", "kMaxGenres", "kWindow", "kMaxMovieSlots",
                 "kIdMask", "kMaxWalkWords"):
        assert isinstance(K.get(name), int) and K[name] > 0, name
    for name in ("kMaxValues", "kMaxProbs", "kMaxBuckets", "kMaxWords", "kMaxTokens", "kMaxWordsPerRow", "kMaxParts",
                 "kMaxMovieId", "kMaxRatings", "kMaxGridBlocks", "kYtyThreads", "kYtyBlocks", "kRankWarps"):
        assert isinstance(K.get(name), int) and K[name] > 0, name
    assert K["kMaxGridBlocks"] == 132 * 64 and K["kMaxTokens"] == (1 << 29) - 1
    assert {constants(f)["kMaxRatings"] for f in RATING_BOUND_FILES} == {MAX_RATINGS}
    assert K["kSrcPerBlock"] == K["kRecWarps"] * K["kSrcPerWarp"]
    assert K["kIdMask"] == K["kMaxMovieSlots"] - 1
    for name in ("kJoinThreads", "kJoinSegments"):
        assert isinstance(K.get(name), int) and K[name] > 0, name
    for name in ("kMaxPairs", "kChunk", "kChunkThreads", "kPerThread", "kMaxGridBlocks"):
        assert isinstance(KB.get(name), int) and KB[name] > 0, name
    assert KB["kPerThread"] * KB["kChunkThreads"] == KB["kChunk"] and KB["kMaxPairs"] == 2 ** 31 - 1
    with pytest.raises(ValueError):                                    # two kChunk: 2 048 points, 32 ratings
        constants("binary_metrics.cu", "als.cu")


def test_vectorised_corpus_matches_chunk_corpus():
    rng = np.random.default_rng(0)
    seqs = [rng.integers(0, 30, n) for n in (1, 999, 1000, 1001, 2500, 3)]
    ids, _ = I.build_vocab(seqs)
    a, b = corpus(seqs, ids), I.chunk_corpus(seqs, ids)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---- rejections one past each bound, before any launch -----------------------------------------------------------
def _p(a):
    return a.ctypes.data


def _i2v_call(vector_size=4, movie=(3, 4, 3), n=None):
    u, m = np.array([1, 1, 2], np.int32), np.array(movie, np.int32)
    h, t = np.array([8, 8, 8], np.int8), np.array([5, 6, 7], np.int32)
    prm = _lib.SrsItem2vecParams(vector_size, 5, 1, 1, 0)
    ids, vec, V = np.zeros(4, np.int32), np.zeros((4, 64), np.float32), C.c_int32(-1)
    if n is not None:
        return _lib.load().srs_item2vec_host(None, None, None, None, n, C.byref(prm), 0, 4, _p(ids), _p(vec),
                                             C.byref(V))
    return _lib.load().srs_item2vec_host(_p(u), _p(m), _p(h), _p(t), 3, C.byref(prm), 0, 4, _p(ids), _p(vec),
                                         C.byref(V))


def _walks_call(num_walks, walk_length):
    u, m = np.array([1, 1], np.int32), np.array([3, 4], np.int32)
    h, t = np.array([8, 8], np.int8), np.array([5, 6], np.int32)
    w, n = np.zeros(1, np.int32), np.zeros(1, np.int32)
    return _lib.load().srs_random_walks_host(_p(u), _p(m), _p(h), _p(t), 2, num_walks, walk_length, 0, 0, _p(w),
                                             _p(n))


def _lsh_call(dim=4, tables=2, k=3):
    x = np.zeros((2, dim), np.float32)
    uv = np.ones((tables, dim)) / np.sqrt(dim)
    keys = np.zeros((1, dim))
    ids, oi, od, oc = np.arange(2, dtype=np.int32), np.zeros(k, np.int32), np.zeros(k), np.zeros(1, np.int32)
    return _lib.load().srs_lsh_query_host(_p(ids), _p(x), 2, dim, _p(uv), tables, 1.0, _p(keys), 1, k, 0, _p(oi),
                                          _p(od), _p(oc))


def _rec_call(rank=3, num=2):
    s, d = np.ones((2, rank), np.float32), np.ones((4, rank), np.float32)
    ids = np.arange(4, dtype=np.int32)
    oi, os_ = np.zeros(2 * max(num, 1), np.int32), np.zeros(2 * max(num, 1), np.float32)
    return _lib.load().srs_als_recommend_host(_p(s), 2, _p(ids), _p(d), 4, rank, num, 0, _p(oi), _p(os_))


def _als_fit_call(rank=3, n=None):
    u, m, r = np.array([1, 2], np.int32), np.array([3, 4], np.int32), np.array([4.0, 5.0], np.float32)
    p = _lib.SrsAlsParams(rank, 1, 0.01, 0)
    ui, mi, uf, mf = np.zeros(2, np.int32), np.zeros(2, np.int32), np.zeros(256, np.float32), np.zeros(256, np.float32)
    nu, nm = C.c_int32(-1), C.c_int32(-1)
    if n is not None:
        return _lib.load().srs_als_fit_host(None, None, None, n, C.byref(p), 0, 2, 2, _p(ui), _p(uf), C.byref(nu),
                                            _p(mi), _p(mf), C.byref(nm))
    return _lib.load().srs_als_fit_host(_p(u), _p(m), _p(r), 2, C.byref(p), 0, 2, 2, _p(ui), _p(uf), C.byref(nu),
                                        _p(mi), _p(mf), C.byref(nm))


def _als_folds_call(n_models, rank=3):
    u, m, r = np.array([1, 2], np.int32), np.array([3, 4], np.int32), np.array([4.0, 5.0], np.float32)
    fold = np.array([0, 1], np.int32)
    specs = (_lib.SrsAlsModel * max(n_models, 1))(*[_lib.SrsAlsModel(rank, 1, 0.01, -1)] * max(n_models, 1))
    M = max(n_models, 1)
    ui, mi = np.zeros(2 * M, np.int32), np.zeros(2 * M, np.int32)
    uf, mf = np.zeros(2 * M * 64, np.float32), np.zeros(2 * M * 64, np.float32)
    nu, nm = np.zeros(M, np.int32), np.zeros(M, np.int32)
    return _lib.load().srs_als_fit_folds_host(_p(u), _p(m), _p(r), _p(fold), 2, 2, specs, n_models, 0, 0, 2, 2,
                                              _p(ui), _p(uf), _p(nu), _p(mi), _p(mf), _p(nm))


def _fe_call(n_genres=1, genres_per_movie=1, n_slots=3, movie=(1, 2, 1), n=None):
    u, m = np.array([1, 1, 1], np.int32), np.array(movie, np.int32)
    h, t = np.array([8, 7, 10], np.int8), np.array([5, 6, 7], np.int32)
    year = np.full(max(n_slots, 1) if n_slots < 100 else 1, 1990, np.int32)
    genres = np.full((len(year), max(genres_per_movie, 1)), -1, np.int32)
    hashes = np.zeros(max(n_genres, 1), np.int32)
    bufs = {f: np.zeros(16, np.int32) for f, _ in _lib.SrsSamples._fields_}
    st = _lib.SrsSamples(**{k: v.ctypes.data for k, v in bufs.items()})
    kept = C.c_int64(-1)
    if n is not None:
        return _lib.load().srs_featureeng_host(None, None, None, None, n, _p(year), _p(genres), n_slots,
                                               genres_per_movie, _p(hashes), n_genres, 0, C.byref(st), C.byref(kept))
    return _lib.load().srs_featureeng_host(_p(u), _p(m), _p(h), _p(t), 3, _p(year), _p(genres), n_slots,
                                           genres_per_movie, _p(hashes), n_genres, 0, C.byref(st), C.byref(kept))


REJECTIONS = {
    "als rank": (lambda: _als_fit_call(rank=K["kMaxRank"] + 1), "rank %d" % (K["kMaxRank"] + 1)),
    "als ratings": (lambda: _als_fit_call(n=MAX_RATINGS + 1), str(MAX_RATINGS)),
    "als folds models": (lambda: _als_folds_call(K["kMaxModels"] + 1), "1..%d" % K["kMaxModels"]),
    "als folds rank": (lambda: _als_folds_call(2, rank=K["kMaxRank"] + 1), "1..%d" % K["kMaxRank"]),
    "als recommend rank": (lambda: _rec_call(rank=K["kMaxRank"] + 1), "1..%d" % K["kMaxRank"]),
    "als recommend num": (lambda: _rec_call(num=K["kMaxNum"] + 1), "1..%d" % K["kMaxNum"]),
    "lsh k": (lambda: _lsh_call(k=K["kMaxK"] + 1), "1..%d" % K["kMaxK"]),
    "lsh dim": (lambda: _lsh_call(dim=K["kMaxLshDim"] + 1), "1..%d" % K["kMaxLshDim"]),
    "lsh tables": (lambda: _lsh_call(tables=K["kMaxTables"] + 1), "1..%d" % K["kMaxTables"]),
    "item2vec dim": (lambda: _i2v_call(vector_size=K["kMaxDim"] + 1), "1..%d" % K["kMaxDim"]),
    "item2vec movie id": (lambda: _i2v_call(movie=(3, K["kMaxMovieSlots"], 3)), "2^24"),
    "item2vec ratings": (lambda: _i2v_call(n=MAX_RATINGS + 1), str(MAX_RATINGS)),
    "walk words": (lambda: _walks_call(K["kMaxWalkWords"] + 1, 1), str(K["kMaxWalkWords"])),
    "walk words product": (lambda: _walks_call((K["kMaxWalkWords"] // 2) + 1, 2), str(K["kMaxWalkWords"])),
    "featureeng genres": (lambda: _fe_call(n_genres=K["kMaxGenres"] + 1), "0..%d" % K["kMaxGenres"]),
    "featureeng genres per movie": (lambda: _fe_call(genres_per_movie=K["kMaxGenres"] + 1), "1..%d" % K["kMaxGenres"]),
    "featureeng slots": (lambda: _fe_call(n_slots=K["kMaxMovieSlots"] + 1), "1..%d" % K["kMaxMovieSlots"]),
    "featureeng movie past the table": (lambda: _fe_call(movie=(1, 3, 1)), "3 slots"),
    "featureeng ratings": (lambda: _fe_call(n=MAX_RATINGS + 1), str(MAX_RATINGS)),
}


@pytest.mark.parametrize("name", sorted(REJECTIONS))
def test_one_past_each_bound_is_rejected_before_any_launch(name):
    from sparrowrecsys_b200.model import launch_count
    call, says = REJECTIONS[name]
    n0 = launch_count()
    rc = call()
    assert rc in (_lib.SRS_ERR_INVALID, _lib.SRS_ERR_RANGE), rc
    msg = _lib.load().srs_last_error().decode()
    assert says in msg, msg
    assert launch_count() == n0


# ---- featurejob.cu and RankingMetrics: one past each bound, before any launch, outputs untouched -----------------
SENTINEL = -7


def _fill(n, t):
    return np.full(max(int(n), 1), SENTINEL, t)


def _quantile_call(n=3, n_probs=2):
    v, p, out = np.array([1.0, 2.0, 3.0]), np.full(max(n_probs, 1), 0.5), _fill(n_probs, np.float64)
    return _lib.load().srs_approx_quantile_host(_p(v) if n <= 3 else None, n, _p(p), n_probs, 0.01, 0,
                                                _p(out)), [out]


def _discretizer_call(n=3, buckets=2):
    v, splits, b, ns = np.array([1.0, 2.0, 3.0]), _fill(K["kMaxBuckets"] + 2, np.float64), _fill(3, np.int32), \
        C.c_int32(SENTINEL)
    rc = _lib.load().srs_quantile_discretizer_host(_p(v) if n <= 3 else None, n, buckets, 0.01, 0, _p(splits),
                                                   C.byref(ns), _p(b))
    return rc, [splits, b, np.array([ns.value])]


def _bucketize_call(n=3, n_splits=3):
    splits = np.r_[-np.inf, np.arange(max(n_splits - 2, 1)), np.inf][:n_splits]
    v, out = np.array([0.5, 1.0, 0.0]), _fill(3, np.int32)
    return _lib.load().srs_bucketize_host(_p(splits), n_splits, _p(v) if n <= 3 else None, n, 0, _p(out)), [out]


def _scale_call(n):
    out, mm = _fill(3, np.float64), _fill(2, np.float64)
    return _lib.load().srs_minmax_scale_host(None, n, None, 0, _p(out), _p(mm)), [out, mm]


def _split_call(n=10, n_parts=2):
    w, rows, cnt = np.ones(n_parts), _fill(10, np.int32), _fill(n_parts, np.int64)
    return _lib.load().srs_sample_split_host(n, 1, 0.5, _p(w), n_parts, 0, _p(rows), _p(cnt)), [rows, cnt]


def _ts_split_call(n=3, ts=(1, 2, 3)):
    t, rows, cnt, split = np.array(ts, np.int64), _fill(3, np.int32), _fill(2, np.int64), C.c_double(SENTINEL)
    rc = _lib.load().srs_sample_split_by_timestamp_host(_p(t) if n <= 3 else None, n, 1, 0.5, 0.01, 0, _p(rows),
                                                        _p(cnt), C.byref(split))
    return rc, [rows, cnt, np.array([split.value])]


def _ratings_call(n=2, movie=(1, 2)):
    m, h = np.array(movie, np.int32), np.array([4, 6], np.int8)
    ids, cnt, avg, var, nm = (_fill(4, np.int32), _fill(4, np.int64), _fill(4, np.float64), _fill(4, np.float64),
                              C.c_int32(SENTINEL))
    rc = _lib.load().srs_rating_features_host(_p(m) if n <= 2 else None, _p(h) if n <= 2 else None, n, 0, 4,
                                              _p(ids), _p(cnt), _p(avg), _p(var), C.byref(nm))
    return rc, [ids, cnt, avg, var, np.array([nm.value])]


def _indexer_call(n_tok=2, W=2, hashes=(1, 2)):
    tok, h = np.array([0, 1], np.int32), np.array(hashes, np.int32)
    lw, lc = _fill(2, np.int32), _fill(2, np.int64)
    rc = _lib.load().srs_string_indexer_host(_p(tok) if n_tok <= 2 else None, n_tok, _p(h), W, 0, _p(lw), _p(lc))
    return rc, [lw, lc]


def _multihot_call(row_len=1, movie=3):
    ids, off = np.array([movie], np.int32), np.array([0, row_len], np.int32)
    words, h = np.zeros(max(row_len, 1), np.int32), np.array([5], np.int32)
    outs = [_fill(1, np.int32), _fill(1, np.int64), _fill(1, np.int32), _fill(2, np.int32), _fill(row_len, np.int32)]
    rc = _lib.load().srs_genre_multihot_host(_p(ids), _p(off), _p(words), 1, _p(h), 1, 0, *[_p(o) for o in outs])
    return rc, outs


def _ranking_call(n_queries, pred_len):
    means = _fill(3, np.float64)
    return _lib.load().srs_ranking_metrics_host(None, n_queries, pred_len, None, None, 5, 0, None, _p(means)), [means]


_VMAX = 2147483647 + 1                          # kMaxValues + 1, checked before any pointer is read
FJ_REJECTIONS = {
    "quantile values": (lambda: _quantile_call(n=_VMAX), "1..%d" % K["kMaxValues"]),
    "discretizer values": (lambda: _discretizer_call(n=_VMAX), "1..%d" % K["kMaxValues"]),
    "bucketize values": (lambda: _bucketize_call(n=_VMAX), "1..%d" % K["kMaxValues"]),
    "scaler values": (lambda: _scale_call(_VMAX), "1..%d" % K["kMaxValues"]),
    "split values": (lambda: _split_call(n=_VMAX), "1..%d" % K["kMaxValues"]),
    "timestamp split values": (lambda: _ts_split_call(n=_VMAX), "1..%d" % K["kMaxValues"]),
    "quantile probabilities": (lambda: _quantile_call(n_probs=K["kMaxProbs"] + 1), "1..%d" % K["kMaxProbs"]),
    "discretizer one bucket": (lambda: _discretizer_call(buckets=1), "2..%d" % K["kMaxBuckets"]),
    "discretizer buckets": (lambda: _discretizer_call(buckets=K["kMaxBuckets"] + 1), "2..%d" % K["kMaxBuckets"]),
    "bucketize splits": (lambda: _bucketize_call(n_splits=K["kMaxBuckets"] + 2), "3..%d" % (K["kMaxBuckets"] + 1)),
    "indexer words": (lambda: _indexer_call(W=K["kMaxWords"] + 1), "1..%d" % K["kMaxWords"]),
    "indexer tokens": (lambda: _indexer_call(n_tok=K["kMaxTokens"] + 1), "1..%d" % K["kMaxTokens"]),
    "indexer hash collision": (lambda: _indexer_call(hashes=(F.java_string_hash("Aa"), F.java_string_hash("BB"))),
                               "share improve(hashCode)"),
    "multi-hot words per row": (lambda: _multihot_call(row_len=K["kMaxWordsPerRow"] + 1),
                                "1..%d" % K["kMaxWordsPerRow"]),
    "multi-hot movie id": (lambda: _multihot_call(movie=K["kMaxMovieId"] + 1), "0..%d" % K["kMaxMovieId"]),
    "rating features movie id": (lambda: _ratings_call(movie=(1, K["kMaxMovieId"] + 1)), "0..%d" % K["kMaxMovieId"]),
    "rating features ratings": (lambda: _ratings_call(n=K["kMaxRatings"] + 1), "1..%d" % K["kMaxRatings"]),
    "split parts": (lambda: _split_call(n_parts=K["kMaxParts"] + 1), "1..%d" % K["kMaxParts"]),
    "timestamp past 2^53": (lambda: _ts_split_call(ts=(0, 2 ** 53 + 1, 5)), "-2^53..2^53"),
    "ranking predictions": (lambda: _ranking_call(1 << 16, 1 << 15), "exceed 2147483647"),
}


@pytest.mark.parametrize("name", sorted(FJ_REJECTIONS))
def test_featurejob_and_ranking_one_past_each_bound_rejected_before_any_launch(name):
    from sparrowrecsys_b200.model import launch_count
    call, says = FJ_REJECTIONS[name]
    n0 = launch_count()
    rc, outs = call()
    assert rc in (_lib.SRS_ERR_INVALID, _lib.SRS_ERR_RANGE), rc
    msg = _lib.load().srs_last_error().decode()
    assert says in msg, msg
    assert launch_count() == n0
    for o in outs:
        assert np.all(o == SENTINEL), (name, o)


def test_the_hash_collision_is_the_oracles_too():
    assert F.java_string_hash("Aa") == F.java_string_hash("BB") == 2112
    with pytest.raises(ValueError):
        FQ.hash_trie_keys(["Aa", "BB"])
    with pytest.raises(ValueError):
        FQ.string_indexer_labels(["Aa", "BB", "Aa"])


# ---- the compress walk's segment cap -----------------------------------------------------------------------------
def _sweep_points():
    rng = np.random.default_rng(56)
    ns = sorted({*range(1, 41), *np.unique(np.geomspace(41, 3e6, 40).astype(int)).tolist(), 3000000})
    eps = [0.0, 1e-7, 1e-6, 1e-5, 1e-4, 2e-4, 5e-4, 1e-3, 1e-2, 0.1, 0.25, 0.5, 0.75, 1.0]
    pts = [(n, e) for n in ns for e in eps]
    pts += [(n, e * x) for n in ns[40::4] for e in (1 / (2 * math.sqrt(n)),) for x in (0.8, 0.9, 0.97, 1.0, 1.1)]
    for _ in range(300):
        n = int(rng.integers(1, 3000001))
        pts.append((n, float(rng.random() / (2 * math.sqrt(n)) * rng.choice([1.0, 2.0]))))
    return pts


def test_the_compress_segments_stay_under_their_cap():
    """fj_compress_kernel's segments under quantiles_of_keys' cap min(n, floor(2 eps n) + 8) + 2, for n from 1 to
    3e6 and eps from 0 to 1 (near 1 / (2 sqrt n) the walk is longest against its cap), plus random draws.  The walk
    takes one segment per run of delta (runs <= 2 eps n + 1) or per head, plus the ends: TIGHT_N, TIGHT_EPS takes
    floor(2 eps n) + 3, the most seen, and the slack of 8 covers it."""
    worst = 0.0
    for n, e in _sweep_points():
        ns, heads = compress_segments(n, e)
        assert ns <= seg_cap(n, e), (n, e, ns)
        assert ns - int(2.0 * e * n) <= 3, (n, e, ns)
        if n <= 20000:
            assert heads == len(FQ.one_summary_closed_form(n, e)) - (n > 1)
        worst = max(worst, ns / seg_cap(n, e))
    ns, _ = compress_segments(TIGHT_N, TIGHT_EPS)
    assert ns - int(2.0 * TIGHT_EPS * TIGHT_N) == 3 and ns / seg_cap(TIGHT_N, TIGHT_EPS) >= worst


def test_the_segment_count_matches_the_oracles_walk():
    for n, e in ((1, 0.0), (2, 0.3), (1000, 0.0), (1000, 0.01), (5000, 0.002), (20001, 0.0035), (77, 1.0)):
        heads = FQ.one_summary_segments(n, e)
        assert compress_segments(n, e)[1] == len(heads) - (n > 1)


def test_vectorised_query_matches_query_sampled():
    rng = np.random.default_rng(57)
    for n, eps in ((1, 0.0), (2, 0.5), (1000, 0.0), (3001, 0.01), (20000, 0.001)):
        v = np.round(rng.standard_normal(n) * 30)
        _, sampled, _ = FQ.one_summary_samples(v, eps)
        p = np.r_[0.0, eps, 1 - eps, 1.0, np.nextafter(eps, 1.0), rng.random(200), np.arange(1, 50) / n]
        p = p[(p >= 0) & (p <= 1)]
        want = [FQ.query_sampled(sampled, n, float(x), eps) for x in p]
        assert query_many(sampled, n, p, eps).tolist() == want
