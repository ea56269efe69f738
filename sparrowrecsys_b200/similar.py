"""Similar movies on the GPU: the reference's SimilarMovieService page, `SimilarMovieProcess.getRecList(movieId,
size, model)` (online/recprocess/SimilarMovieProcess.java:20-32), for many movies per call.

`SimilarMovies(movies, ratings, embeddings)` builds the catalogue once on the device (`srs_similar_catalog_create_host`:
each movie's running-mean rating, each genre's top 100 by rating, the genre masks); `recommend(movie_ids, size,
model)` answers every query in one device call (`srs_similar_movies_host`).  DESIGN.md section 4.23 gives the
semantics; oracle/similar_movies.py restates the Java.

    python -m sparrowrecsys_b200.similar movies.csv ratings.csv [--emb item2vecEmb.csv] [--model emb|default]
        --size N [--all | --movie ID] [--data-manager-rows]
"""
from __future__ import annotations

import ctypes as C
from typing import List, Mapping, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .featureeng import load_movies_csv, load_ratings_csv
from .ranking import load_embeddings_csv

OK, UNKNOWN_MOVIE, NO_EMBEDDING = _lib.SRS_SIMILAR_OK, _lib.SRS_SIMILAR_UNKNOWN_MOVIE, _lib.SRS_SIMILAR_NO_EMBEDDING
STATUS_NAMES = {OK: "ok", UNKNOWN_MOVIE: "unknown movie", NO_EMBEDDING: "missing embedding"}
_JAVA_WS = "".join(chr(c) for c in range(33))          # java.lang.String.trim strips every char <= ' '


class SimilarList(NamedTuple):
    movie_ids: np.ndarray      # int32, best first
    scores: np.ndarray         # float64
    status: int                # OK, UNKNOWN_MOVIE or NO_EMBEDDING


def java_split(s: str, sep: str) -> List[str]:
    """String.split(sep) for a one-character separator: trailing empty strings removed."""
    parts = s.split(sep)
    while parts and parts[-1] == "":
        parts.pop()
    return parts if parts else [""] if s == "" else parts


def genre_lists(genres: Sequence[str]) -> List[List[str]]:
    """DataManager.loadMovieData's genres: none when the field is blank, else String.split("\\\\|")."""
    return [[] if g.strip(_JAVA_WS) == "" else java_split(g, "|") for g in genres]


def data_manager_rows(path: str) -> np.ndarray:
    """The movie ids DataManager.loadMovieData keeps from movies.csv: the lines (after the header) whose
    String.split(",") has exactly three fields.  A title with a comma (quoted in the CSV) makes more fields, so the
    reference's server does not know that movie."""
    ids = []
    with open(path, encoding="utf-8") as f:
        next(f, None)
        for line in f:
            parts = java_split(line.rstrip("\r\n"), ",")
            if len(parts) == 3:
                ids.append(int(parts[0]))
    return np.asarray(ids, np.int32)


class SimilarMovies:
    """The similar-movies catalogue on one device.

    `movies`: movieId and genres in movies.csv order (as `featureeng.load_movies_csv` returns); `ratings`: movieId and
    rating in ratings.csv order (as `featureeng.load_ratings_csv`); `embeddings`: the (ids, vectors [n, dim]) of
    `ranking.load_embeddings_csv`, or None.  Movie ids must be distinct, a movie must not list a genre twice, and
    there may be at most 64 distinct genres; a violation raises ValueError before any device work."""

    def __init__(self, movies: Mapping[str, object], ratings: Mapping[str, np.ndarray],
                 embeddings: Optional[Tuple[np.ndarray, np.ndarray]] = None, device: int = 0):
        ids = np.ascontiguousarray(movies["movieId"], np.int32)
        lists = genre_lists(list(movies["genres"]))
        if len(lists) != ids.shape[0]:
            raise ValueError("movies: %d ids but %d genre fields" % (ids.shape[0], len(lists)))
        vocab = {}
        flat = [vocab.setdefault(g, len(vocab)) for gl in lists for g in gl]
        self.genres = list(vocab)
        off = np.zeros(len(lists) + 1, np.int32)
        off[1:] = np.cumsum([len(gl) for gl in lists])
        genre = np.asarray(flat or [0], np.int32)
        rmovie = np.ascontiguousarray(ratings["movieId"], np.int32)
        rscore = np.ascontiguousarray(ratings["rating"], np.float32)       # Float.parseFloat
        if rmovie.shape != rscore.shape:
            raise ValueError("ratings: movieId and rating differ in length")
        if embeddings is None:
            eid, emb, dim = np.zeros(1, np.int32), np.zeros(1, np.float32), 0
            n_emb = 0
        else:
            eid = np.ascontiguousarray(embeddings[0], np.int32)
            emb = np.ascontiguousarray(embeddings[1], np.float32)
            if emb.ndim != 2 or emb.shape[0] != eid.shape[0] or (eid.shape[0] and emb.shape[1] < 1):
                raise ValueError("embeddings: ids [n] and vectors [n, dim >= 1] expected, got %s and %s"
                                 % (eid.shape, emb.shape))
            n_emb, dim = eid.shape[0], (emb.shape[1] if eid.shape[0] else 0)
        self.device = device
        self.dim = dim
        lib = _lib.load()
        h = C.c_void_p()
        p = lambda a: a.ctypes.data
        _lib.check(lib.srs_similar_catalog_create_host(p(ids), ids.shape[0], p(off), p(genre), len(vocab), p(rmovie),
                                                       p(rscore), rmovie.shape[0], p(eid), p(emb), n_emb, dim, device,
                                                       C.byref(h)))
        self._h = h

    def close(self) -> None:
        if getattr(self, "_h", None):
            _lib.load().srs_similar_catalog_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def recommend_arrays(self, movie_ids, size: int, model: str = "emb"):
        """One device call for every query: (ids int32 [Q, size], scores float64 [Q, size], count int32 [Q],
        status int32 [Q]); row q's first count[q] entries are its list, the rest 0.  `model` "emb" is the cosine
        ranker, any other string calculateSimilarScore, as the Java's switch."""
        if self._h is None:
            raise ValueError("the catalogue is closed")
        q = np.ascontiguousarray(movie_ids, np.int32).reshape(-1)
        size = int(size)
        if size < 1:
            raise ValueError("size must be >= 1, got %d" % size)
        Q = q.shape[0]
        ids = np.zeros((Q, size), np.int32)
        scores = np.zeros((Q, size), np.float64)
        count = np.zeros(Q, np.int32)
        status = np.zeros(Q, np.int32)
        m = _lib.SRS_SIMILAR_EMB if model == "emb" else _lib.SRS_SIMILAR_DEFAULT
        p = lambda a: a.ctypes.data
        _lib.check(_lib.load().srs_similar_movies_host(self._h, p(q), Q, size, m, p(ids), p(scores), p(count),
                                                       p(status)))
        return ids, scores, count, status

    def recommend(self, movie_ids, size: int, model: str = "emb") -> List[SimilarList]:
        """getRecList(movie_id, size, model) for each of `movie_ids`."""
        ids, scores, count, status = self.recommend_arrays(movie_ids, size, model)
        return [SimilarList(ids[i, :count[i]].copy(), scores[i, :count[i]].copy(), int(status[i]))
                for i in range(ids.shape[0])]


def main(argv: Sequence[str]) -> int:
    import argparse
    ap = argparse.ArgumentParser(prog="python -m sparrowrecsys_b200.similar")
    ap.add_argument("movies")
    ap.add_argument("ratings")
    ap.add_argument("--emb", help="item2vecEmb.csv: id:v v v ... lines")
    ap.add_argument("--model", default="emb", choices=("emb", "default"))
    ap.add_argument("--size", type=int, required=True)
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument("--all", action="store_true", help="every movie of the catalogue, in movies.csv order")
    g.add_argument("--movie", type=int)
    ap.add_argument("--data-manager-rows", action="store_true",
                    help="keep only the movies.csv lines the reference's DataManager loads (no comma in the title)")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    movies = load_movies_csv(a.movies)
    if a.data_manager_rows:
        keep = np.isin(movies["movieId"], data_manager_rows(a.movies))
        movies = {"movieId": movies["movieId"][keep], "genres": [x for x, k in zip(movies["genres"], keep) if k]}
    ratings = load_ratings_csv(a.ratings)
    emb = load_embeddings_csv(a.emb) if a.emb else None
    if a.model == "emb" and emb is None:
        ap.error("--model emb needs --emb")
    queries = movies["movieId"] if a.all else np.array([a.movie], np.int32)
    with SimilarMovies(movies, ratings, emb, a.device) as s:
        for mid, r in zip(np.asarray(queries).tolist(), s.recommend(queries, a.size, a.model)):
            if r.status != OK:
                print("%d\t(%s)" % (mid, STATUS_NAMES[r.status]))
            else:
                print("%d\t%s" % (mid, " ".join("%d:%.17g" % (i, x) for i, x in zip(r.movie_ids.tolist(),
                                                                                    r.scores.tolist()))))
    return 0


if __name__ == "__main__":
    import sys
    sys.exit(main(sys.argv[1:]))
