"""SimilarMovieProcess's two other candidate sources restated literally in Python, on top of oracle/similar_movies.py:
`multipleRetrievalCandidates` (online/recprocess/SimilarMovieProcess.java:56-83) and
`retrievalCandidatesByEmbedding` (:91-112).

* `DataManager.parseReleaseYear` (DataManager.java:167-178) on the trimmed title field: `substring(len - 5,
  len - 1)` through `Integer.parseInt`; -1 when the title is shorter than 6 characters or the parse fails, and
  loadMovieData then leaves `releaseYear` at 0.  A parsed -1 is indistinguishable from a failure and also gives 0.
* `getMovies(size, sortBy)` (:271-283): a stable sort of `new ArrayList<>(movieMap.values())`.  movieMap is a
  `HashMap<Integer, Movie>` filled in load order, so ties come out in its iteration order: buckets
  `(id ^ (id >>> 16)) & (capacity - 1)` ascending, load order within a bucket (`hashmap_order` simulates the puts).
* Multi-channel recall: the union of each genre's `getMoviesByGenre(genre, 20, "rating")`, `getMovies(100,
  "rating")` and `getMovies(100, "releaseYear")`, minus the query; ranked as `getRecList` ranks the genre candidates.
* Embedding recall: `getMovies(10000, "rating")`, the query included, scored by `calculateEmbSimilarScore` (-1 for a
  movie without a vector), sorted by `Map.Entry.comparingByValue()`: ascending `Double.compare`, so -1s first and
  NaN last - the least similar movies.  Java leaves ties in identity-hash order; here they go by movie id.
"""
from __future__ import annotations

import functools

import numpy as np

from . import similar_movies as S
from .ctr_oracle import java_double_compare

MULTI_GENRE_TOP, GLOBAL_TOP, POOL = 20, 100, 10000
_JAVA_WS = "".join(chr(c) for c in range(33))          # String.trim strips every char <= ' '


class TreeifiedBin(ValueError):
    """A put would turn a HashMap bin into a tree, whose iteration order is no longer load order."""


def java_parse_int(s: str) -> int:
    """Integer.parseInt(s): an optional '+' or '-', then one or more decimal digits (any Unicode Nd digit, as
    Character.digit takes), within the int range; anything else raises ValueError (NumberFormatException)."""
    body = s[1:] if s[:1] in ("+", "-") else s
    if not body or not all(c.isdecimal() for c in body):
        raise ValueError("not an int: %r" % (s,))
    v = int(("-" if s[:1] == "-" else "") + "".join(str(int(c)) for c in body))
    if not -2 ** 31 <= v < 2 ** 31:
        raise ValueError("out of int range: %r" % (s,))
    return v


def parse_release_year(title) -> int:
    """The releaseYear loadMovieData gives a movie from its title field (movieData[1]): parseReleaseYear of the trimmed
    field, in UTF-16 code units as Java indexes strings, and 0 where that returns -1.  Unlike
    `featureeng.release_year` there is no 1990 default and no exception."""
    if title is None:
        return 0
    t = title.strip(_JAVA_WS)
    u = t.encode("utf-16-le", "surrogatepass")
    n = len(u) // 2
    if n < 6:
        return 0
    try:
        y = java_parse_int(u[2 * (n - 5):2 * (n - 1)].decode("utf-16-le", "surrogatepass"))
    except (ValueError, UnicodeDecodeError):
        return 0
    return 0 if y == -1 else y


def _spread(i: int) -> int:
    h = i & 0xFFFFFFFF
    return h ^ (h >> 16)


def hashmap_order(ids):
    """(iteration order as load indices, table length) of a java.util.HashMap<Integer, _> after put(ids[0]), ...,
    put(ids[n-1]) (distinct keys), simulated put by put as JDK 8's putVal / resize / treeifyBin do it.  Raises
    TreeifiedBin where a put makes a bin's ninth entry in a table of 64 or more."""
    cap, table = 16, [[] for _ in range(16)]

    def resize():
        nonlocal cap, table
        cap *= 2
        new = [[] for _ in range(cap)]
        for b in table:                      # the split keeps each bucket's relative order
            for i in b:
                new[_spread(ids[i]) & (cap - 1)].append(i)
        table = new

    ids = [int(x) for x in ids]
    for i, key in enumerate(ids):
        b = table[_spread(key) & (cap - 1)]
        b.append(i)
        if len(b) > 8:                       # binCount >= TREEIFY_THRESHOLD - 1
            if cap >= 64:
                raise TreeifiedBin("movie id %d makes a 9th entry in a bucket of a %d-bucket table" % (key, cap))
            resize()                         # MIN_TREEIFY_CAPACITY: treeifyBin resizes instead
        if i + 1 > cap * 3 // 4:             # ++size > threshold
            resize()
    return [i for b in table for i in b], cap


class RecallCatalogue(S.Catalogue):
    """oracle/similar_movies.Catalogue plus each movie's release year (`release_year`, in load order, as
    `parse_release_year` gives it; None for none) and DataManager.getMovies."""

    def __init__(self, movie_ids, genres, rating_movie, rating_score, emb_ids=None, emb=None, release_year=None,
                 cosine=S.java_cosine_many):
        super().__init__(movie_ids, genres, rating_movie, rating_score, emb_ids, emb, cosine)
        self.year = None if release_year is None else [int(y) for y in release_year]
        self._sorted = {}

    def get_movies(self, size, sort_by):
        """getMovies(size, sortBy), as slots; raises TreeifiedBin where movieMap's order is not restated."""
        if sort_by not in self._sorted:
            lst = hashmap_order(self.ids)[0]
            if sort_by == "rating":
                lst.sort(key=functools.cmp_to_key(lambda a, b: java_double_compare(self.avg[b], self.avg[a])))
            elif sort_by == "releaseYear":
                y = self.year
                lst.sort(key=functools.cmp_to_key(lambda a, b: (y[b] > y[a]) - (y[b] < y[a])))
            self._sorted[sort_by] = lst
        return self._sorted[sort_by][:size]

    def multiple_candidates(self, m):
        """multipleRetrievalCandidates(movie), as a set of slots (the Java's list order is its HashMap's)."""
        cands = set()
        for g in set(self.genres[m]):
            cands.update(self.movies_by_genre(g, MULTI_GENRE_TOP))
        cands.update(self.get_movies(GLOBAL_TOP, "rating"))
        cands.update(self.get_movies(GLOBAL_TOP, "releaseYear"))
        cands.discard(m)
        return sorted(cands)

    def rec_list(self, movie_id, size, model="emb", candidates="genre"):
        """(ids, scores, status) of getRecList(movie_id, size, model) with `candidates` "genre"
        (candidateGenerator) or "multiple" (multipleRetrievalCandidates)."""
        if candidates == "genre":
            return super().rec_list(movie_id, size, model)
        if candidates != "multiple":
            raise ValueError("candidates must be 'genre' or 'multiple', got %r" % (candidates,))
        m = self.slot.get(int(movie_id))
        if m is None:
            return [], [], S.UNKNOWN_MOVIE
        if model == "emb" and m not in self.emb:
            return [], [], S.NO_EMBEDDING
        cands = self.multiple_candidates(m)
        if model == "emb":
            have = [c for c in cands if c in self.emb]
            s = dict(zip(have, self.cosine(self.emb[m], np.array([self.emb[c] for c in have]))
                         if have else []))
            scores = [float(s[c]) if c in s else -1.0 for c in cands]
        else:
            scores = [self.similar_score(m, c) for c in cands]
        items = sorted(((scores[i], self.ids[c]) for i, c in enumerate(cands)),
                       key=functools.cmp_to_key(lambda x, y: java_double_compare(y[0], x[0]) or
                                                (x[1] > y[1]) - (x[1] < y[1])))[:size]
        return [i for _, i in items], [s for s, _ in items], S.OK

    def embedding_recall(self, movie_id, size):
        """(ids, scores, status) of retrievalCandidatesByEmbedding(movie, size)."""
        m = self.slot.get(int(movie_id))
        if m is None:
            return [], [], S.UNKNOWN_MOVIE
        if m not in self.emb:
            return [], [], S.NO_EMBEDDING
        pool = self.get_movies(POOL, "rating")
        have = [c for c in pool if c in self.emb]
        s = dict(zip(have, self.cosine(self.emb[m], np.array([self.emb[c] for c in have]))
                     if have else []))
        items = sorted(((float(s[c]) if c in s else -1.0, self.ids[c]) for c in pool),
                       key=functools.cmp_to_key(lambda x, y: java_double_compare(x[0], y[0]) or
                                                (x[1] > y[1]) - (x[1] < y[1])))[:size]
        return [i for _, i in items], [s for s, _ in items], S.OK
