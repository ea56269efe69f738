"""SimilarMovieProcess.getRecList (online/recprocess/SimilarMovieProcess.java:20-32) restated literally in Python.

* `DataManager.loadMovieData` / `loadRatingData` / `loadMovieEmb`: movies in file order, each genre's reverse-index
  list in load order, `Movie.addRating`'s running mean in float64 over the ratings in file order (Movie.java:93-95),
  the last vector line of a movie winning.
* `getMoviesByGenre(genre, 100, "rating")` (DataManager.java:253-268): a stable sort of a copy of the genre's list
  by `Double.compare(m2.avg, m1.avg)`, first 100.
* `candidateGenerator` (:39-49): the union of those lists over the movie's genres, minus the movie.
* `calculateSimilarScore` (:145-159) in float64 - NaN, the Java's `(double) 0 / 0`, when neither movie has a genre -
  or `Embedding.calculateSimilarity` (Embedding.java:33-47): float products summed in double in index order; a
  candidate without a vector scores -1.  `cosine` (a constructor argument) sums in that order by default;
  `warp_cosine_many` restates the device's lane order (csrc/cosine.cuh), which can differ in the last bit.
* The ranking sorts by `Double.compare` descending; Java leaves tied scores in HashMap order, here they go by movie
  id ascending.
Status: OK, UNKNOWN_MOVIE (empty list, as the Java), NO_EMBEDDING (the Java throws a NullPointerException on a query
movie without a vector under "emb"; here that query has an empty list).
"""
from __future__ import annotations

import functools

import numpy as np

from .ctr_oracle import java_double_compare

OK, UNKNOWN_MOVIE, NO_EMBEDDING = 0, 1, 2
GENRE_TOP = 100


def running_mean(scores) -> float:
    """Movie.addRating's averageRating after `scores` (float32 values, file order)."""
    avg, n = 0.0, 0
    for s in scores:
        avg = (avg * n + float(np.float32(s))) / (n + 1)
        n += 1
    return avg


def java_cosine(a, b) -> float:
    """Embedding.calculateSimilarity: float products accumulated in double in index order."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    dot = d1 = d2 = 0.0
    for x, y in zip(a, b):
        dot += float(x * y)
        d1 += float(x * x)
        d2 += float(y * y)
    return dot / (np.sqrt(d1) * np.sqrt(d2))


def java_cosine_many(q, C):
    """java_cosine(q, C[i]) for every row, vectorised over rows (the sum over the index stays sequential)."""
    q = np.asarray(q, np.float32)
    C = np.asarray(C, np.float32).reshape(-1, q.shape[0])
    dot = np.zeros(C.shape[0])
    d2 = np.zeros(C.shape[0])
    d1 = 0.0
    for i in range(q.shape[0]):
        dot += (q[i] * C[:, i]).astype(np.float64)
        d2 += (C[:, i] * C[:, i]).astype(np.float64)
        d1 += float(q[i] * q[i])
    with np.errstate(divide="ignore", invalid="ignore"):
        return dot / (np.sqrt(d1) * np.sqrt(d2))


def _warp_sum(P):
    """csrc/cosine.cuh's sum of each row of the float64 products P [n, dim]: lane l sums elements l, l + 32, ... in
    order from +0.0, then an xor tree over offsets 16, 8, 4, 2, 1 (lane l adds lane l ^ o); every lane ends equal."""
    s = np.zeros((P.shape[0], 32))
    for k in range(0, P.shape[1], 32):
        w = min(32, P.shape[1] - k)
        s[:, :w] += P[:, k:k + w]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lanes ^ o]
    return s[:, 0]


def warp_cosine_many(q, C):
    """The device's cosine of q and each row of C (csrc/cosine.cuh, one warp per pair): float products widened to
    double, summed in lane order (`_warp_sum`), dot / (sqrt(n1) * sqrt(n2)).  The same bits as `java_cosine_many`
    whenever the sums are exact; otherwise they may differ in the last bit."""
    q = np.asarray(q, np.float32)
    C = np.asarray(C, np.float32).reshape(-1, q.shape[0])
    dot = _warp_sum((q[None, :] * C).astype(np.float64))
    d2 = _warp_sum((C * C).astype(np.float64))
    d1 = _warp_sum((q * q).astype(np.float64)[None, :])[0]
    with np.errstate(divide="ignore", invalid="ignore"):
        return dot / (np.sqrt(d1) * np.sqrt(d2))


class Catalogue:
    """movie_ids in movies.csv order, genres[m] the list of movie m's genre strings, the ratings (movie id, score)
    in ratings.csv order, and optionally the vector file's (ids, vectors) rows.  `cosine(q, C)` scores the emb
    ranker: `java_cosine_many` (the Java's order) or `warp_cosine_many` (the device's)."""

    def __init__(self, movie_ids, genres, rating_movie, rating_score, emb_ids=None, emb=None,
                 cosine=java_cosine_many):
        self.cosine = cosine
        self.ids = [int(x) for x in movie_ids]
        self.genres = [list(g) for g in genres]
        self.slot = {}
        for m, i in enumerate(self.ids):
            if i in self.slot:
                raise ValueError("movie id %d appears twice" % i)
            self.slot[i] = m
        self.index = {}
        for m, gl in enumerate(self.genres):
            for g in gl:
                self.index.setdefault(g, []).append(m)
        per_movie = [[] for _ in self.ids]
        for mid, s in zip(np.asarray(rating_movie).tolist(), np.asarray(rating_score, np.float32).tolist()):
            m = self.slot.get(int(mid))
            if m is not None:
                per_movie[m].append(s)
        self.avg = [running_mean(s) for s in per_movie]
        self.emb = {}
        if emb_ids is not None:
            for i, v in zip(np.asarray(emb_ids).tolist(), np.asarray(emb, np.float32)):
                m = self.slot.get(int(i))
                if m is not None:
                    self.emb[m] = v
        self._by_genre = {}

    def movies_by_genre(self, genre, size=GENRE_TOP):
        """getMoviesByGenre(genre, size, "rating"), as slots."""
        if genre not in self._by_genre:
            lst = list(self.index[genre])
            lst.sort(key=functools.cmp_to_key(lambda a, b: java_double_compare(self.avg[b], self.avg[a])))
            self._by_genre[genre] = lst
        return self._by_genre[genre][:size]

    def candidates(self, m):
        seen = {}
        for g in self.genres[m]:
            for c in self.movies_by_genre(g):
                seen[c] = True
        seen.pop(m, None)
        return list(seen)

    def similar_score(self, m, c):
        same = sum(1 for g in self.genres[m] if g in self.genres[c])
        sizes = len(self.genres[m]) + len(self.genres[c])
        genre_similarity = same / sizes / 2 if sizes else float("nan")     # Java's (double) 0 / 0
        rating_score = self.avg[c] / 5
        return genre_similarity * 0.7 + rating_score * 0.3

    def rec_list(self, movie_id, size, model="emb"):
        """(ids, scores, status) of getRecList(movie_id, size, model)."""
        m = self.slot.get(int(movie_id))
        if m is None:
            return [], [], UNKNOWN_MOVIE
        if model == "emb" and m not in self.emb:
            return [], [], NO_EMBEDDING
        cands = self.candidates(m)
        if model == "emb":
            have = [c for c in cands if c in self.emb]
            s = dict(zip(have, self.cosine(self.emb[m], np.array([self.emb[c] for c in have]))
                         if have else []))
            scores = [float(s[c]) if c in s else -1.0 for c in cands]
        else:
            scores = [self.similar_score(m, c) for c in cands]
        items = [(scores[i], self.ids[c]) for i, c in enumerate(cands)]

        def order(x, y):
            r = java_double_compare(y[0], x[0])
            return r if r else (x[1] > y[1]) - (x[1] < y[1])
        items.sort(key=functools.cmp_to_key(order))
        items = items[:size]
        return [i for _, i in items], [s for s, _ in items], OK
