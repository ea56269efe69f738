"""numpy restatement of the reference's DeepWalk graph embedding (Embedding.scala:140-228, 254-266): the item
transition matrix of consecutive positive ratings, random walks over it, and Word2Vec over the walks.

THIS IS THE READABLE SPEC, NOT PRODUCT.  The walks use the library's draws, so the tests hold the device to these
walks exactly; the Word2Vec part is `oracle/item2vec_c.c` run on them.  DESIGN.md section 4.14 gives the semantics
and the orders Scala leaves open.
"""
from __future__ import annotations

import numpy as np

from . import item2vec as I

_M64 = (1 << 64) - 1
_GOLDEN = 0x9E3779B97F4A7C15


def pairs(seqs):
    """Every consecutive (s[i], s[i + 1]) within a sentence: (a int64 [N], b int64 [N]), in corpus order."""
    a = [s[:-1] for s in seqs if len(s) > 1]
    b = [s[1:] for s in seqs if len(s) > 1]
    if not a:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(a).astype(np.int64), np.concatenate(b).astype(np.int64)


def transitions(seqs):
    """generateTransitionMatrix with sources and each row's targets ascending.  Returns a dict: sources [S],
    out [S] = out(a), dist [S] = out(a) / pairTotal, cdf [S] (its cumulative sums), row_ptr [S + 1], targets [E],
    counts [E], probs [E] = count / out(a), cum [E] (each row's cumulative sums).  Every probability is one double
    division and every cumulative sum adds left to right (np.cumsum accumulates sequentially)."""
    a, b = pairs(seqs)
    key, counts = np.unique(a * (1 << 24) + b, return_counts=True)
    src, tgt = key >> 24, key & ((1 << 24) - 1)
    starts = np.flatnonzero(np.r_[True, src[1:] != src[:-1]]) if len(key) else np.zeros(0, np.int64)
    row_ptr = np.r_[starts, len(key)].astype(np.int64)
    out = np.add.reduceat(counts, starts) if len(key) else np.zeros(0, np.int64)
    row_of_entry = np.repeat(np.arange(len(starts)), np.diff(row_ptr))
    probs = counts.astype(np.float64) / out[row_of_entry].astype(np.float64)
    cum = np.empty_like(probs)
    for r in range(len(starts)):
        lo, hi = row_ptr[r], row_ptr[r + 1]
        cum[lo:hi] = np.cumsum(probs[lo:hi])
    total = int(out.sum())
    dist = out.astype(np.float64) / float(total) if total else np.zeros(0)
    return {"sources": src[starts], "out": out.astype(np.int64), "dist": dist, "cdf": np.cumsum(dist),
            "row_ptr": row_ptr, "targets": tgt, "counts": counts.astype(np.int64), "probs": probs, "cum": cum}


def _splitmix(x, i):
    """item2vec's splitmix over uint64 arrays: splitmix64's finaliser of x + (i + 1) * golden (mod 2^64)."""
    with np.errstate(over="ignore"):
        z = np.asarray(x, np.uint64) + (np.asarray(i, np.uint64) + np.uint64(1)) * np.uint64(_GOLDEN)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def walk_uniforms(seed, w, t):
    """u of walks w (array) at step t: the top 53 bits of splitmix(splitmix(splitmix(~seed, 0), w), t) over 2^53.
    Word2Vec's windows use splitmix(~seed, k) for iterations k >= 1, so key 0 is the walks' own stream."""
    root = I.splitmix(~int(seed) & _M64, 0)
    h = _splitmix(_splitmix(np.uint64(root), np.asarray(w, np.uint64)), np.uint64(t))
    return (h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def _first_at_least(cum, lo, hi, u):
    """Per walk, the first entry e in [lo, hi) with cum[e] >= u (hi if none): a vectorised binary search."""
    lo, hi = lo.copy(), hi.copy()
    end = hi.copy()
    while True:
        open_ = lo < hi
        if not open_.any():
            return np.where(lo < end, lo, end)
        mid = (lo + hi) // 2
        ok = np.zeros(len(lo), bool)
        ok[open_] = cum[mid[open_]] >= u[open_]
        hi = np.where(open_ & ok, mid, hi)
        lo = np.where(open_ & ~ok, mid + 1, lo)


def random_walks(tr, num_walks, walk_length, seed=0, uniforms=None):
    """randomWalk: (walks int32 [W][L], -1 past each walk's end; lengths int32 [W]).  `uniforms(w, t)` (default
    `walk_uniforms` of `seed`) gives the draws of walks w at step t.  The first item comes from dist; a u past the
    last cumulative sum leaves an empty walk.  Later steps stop at an item with no outgoing pair; a u past its row's
    last sum repeats the current item."""
    u_of = uniforms or (lambda w, t: walk_uniforms(seed, w, t))
    W, L = int(num_walks), int(walk_length)
    walks = np.full((W, L), -1, np.int32)
    lengths = np.zeros(W, np.int32)
    S = len(tr["sources"])
    w = np.arange(W)
    r0 = np.searchsorted(tr["cdf"], u_of(w, 0), side="left")       # the first index with cdf >= u
    alive = r0 < S
    cur = np.where(alive, tr["sources"][np.minimum(r0, max(S - 1, 0))] if S else 0, -1)
    walks[alive, 0] = cur[alive]
    lengths[alive] = 1
    top = max([int(tr["sources"].max()) if S else 0] + [int(tr["targets"].max()) if len(tr["targets"]) else 0])
    row_of = np.full(top + 2, -1, np.int64)
    row_of[tr["sources"]] = np.arange(S)
    for t in range(1, L):
        alive = alive & (row_of[cur] >= 0)
        if not alive.any():
            break
        idx = np.flatnonzero(alive)
        r = row_of[cur[idx]]
        lo, hi = tr["row_ptr"][r], tr["row_ptr"][r + 1]
        e = _first_at_least(tr["cum"], lo, hi, u_of(idx, t))
        nxt = np.where(e < hi, tr["targets"][np.minimum(e, len(tr["targets"]) - 1)], cur[idx])
        cur[idx] = nxt
        walks[idx, t] = nxt
        lengths[idx] += 1
    return walks, lengths


def walk_sentences(walks, lengths):
    """The non-empty walks as Word2Vec sentences (int64 arrays)."""
    return [walks[i, :lengths[i]].astype(np.int64) for i in range(len(lengths)) if lengths[i] > 0]


def graph_embedding(user, movie, half, ts, vector_size=10, window=5, iterations=10, partitions=1, seed=0,
                    num_walks=20000, walk_length=10):
    """graphEmb: ratings -> (vocabulary ids [V], vectors [V][vector_size]), Word2Vec in C (oracle/item2vec_c.c)."""
    from . import item2vec_cext as X
    _, seqs = I.positive_sequences(user, movie, half, ts)
    walks, lengths = random_walks(transitions(seqs), num_walks, walk_length, seed)
    sents = walk_sentences(walks, lengths)
    ids, counts = I.build_vocab(sents)
    words, offs = I.chunk_corpus(sents, ids)
    code, point, codelen = I.huffman(counts)
    return ids, X.train(words, offs, counts, code, point, codelen, vector_size, window, iterations, partitions, seed)
