"""The offline jobs at their bounds and tile edges (csrc/item2vec.cu, graphemb.cu, lsh.cu, als.cu, featureeng.cu).

`BOUNDS` names one case per (job, edge).  Each case builds its inputs here; its `reach` shows from the oracle alone,
with no device, that the inputs reach the edge the case names, and returns the (bound, value) pairs it reaches.
tests/test_gpu_offline_bounds.py runs every case on the device against its oracle, bit for bit, twice.

The bounds come from the kernels' own constants: `test_every_bound_has_a_case` parses them, so a changed constant
without a case at its new value fails.  The size bounds (21 000 000 ratings, kMaxWalkWords) are covered by the
rejection one past them; the deepest Huffman case is the largest run.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import re
from typing import Callable, NamedTuple

import numpy as np
import pytest

from oracle import als as A
from oracle import feature_eng as F
from oracle import graphemb as G
from oracle import item2vec as I
from oracle import lsh as H
from sparrowrecsys_b200 import _lib

from test_item2vec_oracle import MAX_RATINGS, _deepest_counts

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc")


# ---- the kernels' constants --------------------------------------------------------------------------------------
def constants(*files):
    """name -> value of every `constexpr` integer in the given csrc files (simple integer expressions)."""
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
                out[name] = int(eval(e, {"__builtins__": {}}))
            except (NameError, SyntaxError):
                pass
    return out


K = constants("als.cu", "lsh.cu", "item2vec.cu", "featureeng.cu", "graphemb.cu")


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
    assert need <= have, sorted(need - have)
    # the deepest case is the deepest code the rating bound allows: one level more needs more ratings than it takes
    assert sum(_deepest_counts(DEEPEST + 1)) > MAX_RATINGS >= sum(_deepest_counts(DEEPEST))
    assert DEEPEST < K["kMaxCode"]


def test_the_constants_are_parsed():
    for name in ("kMaxRank", "kMaxNum", "kTile", "kChunk", "kSrcPerBlock", "kMaxModels", "kMaxK", "kMaxLshDim",
                 "kMaxTables", "kQueryWarps", "kMaxCode", "kMaxDim", "kMaxGenres", "kWindow", "kMaxMovieSlots",
                 "kIdMask", "kMaxWalkWords"):
        assert isinstance(K.get(name), int) and K[name] > 0, name
    assert K["kSrcPerBlock"] == K["kRecWarps"] * K["kSrcPerWarp"]
    assert K["kIdMask"] == K["kMaxMovieSlots"] - 1


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
