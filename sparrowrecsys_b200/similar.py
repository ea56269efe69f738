"""Similar movies on the GPU: the reference's SimilarMovieService page, `SimilarMovieProcess.getRecList(movieId,
size, model)` (online/recprocess/SimilarMovieProcess.java:20-32), for many movies per call.

`SimilarMovies(movies, ratings, embeddings)` builds the catalogue once on the device
(`srs_similar_catalog_create_ex_host`: each movie's running-mean rating, each genre's top 100 by rating, the genre
masks, and DataManager.getMovies' top lists by rating and release year); `recommend(movie_ids, size, model,
candidates)` answers every query in one device call (`srs_similar_movies_candidates_host`), with the genre candidates
of `candidateGenerator` or the multi-channel recall of `multipleRetrievalCandidates`, and
`retrieve_by_embedding(movie_ids, size)` is `retrievalCandidatesByEmbedding` (`srs_similar_embedding_recall_host`).
DESIGN.md sections 4.23 and 4.24 give the semantics; oracle/similar_movies.py and oracle/similar_recall.py restate
the Java.

    python -m sparrowrecsys_b200.similar movies.csv ratings.csv [--emb item2vecEmb.csv] [--model emb|default]
        [--candidates genre|multiple | --embedding-recall] --size N [--all | --movie ID] [--data-manager-rows]
"""
from __future__ import annotations

import ctypes as C
import re
from typing import List, Mapping, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .featureeng import load_movies_csv, load_ratings_csv
from .ranking import load_embeddings_csv

OK, UNKNOWN_MOVIE, NO_EMBEDDING = _lib.SRS_SIMILAR_OK, _lib.SRS_SIMILAR_UNKNOWN_MOVIE, _lib.SRS_SIMILAR_NO_EMBEDDING
STATUS_NAMES = {OK: "ok", UNKNOWN_MOVIE: "unknown movie", NO_EMBEDDING: "missing embedding"}
_JAVA_WS = "".join(chr(c) for c in range(33))          # java.lang.String.trim strips every char <= ' '
_JAVA_INT = re.compile(r"[+-]?[0-9]+")                  # Integer.parseInt of ASCII text


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


def data_manager_release_year(title: Optional[str]) -> int:
    """Movie.releaseYear as DataManager.loadMovieData sets it from a title field: parseReleaseYear
    (DataManager.java:167-178) takes the trimmed field's UTF-16 code units [len - 5, len - 1) through
    Integer.parseInt (an optional sign, then decimal digits); where the field is shorter than 6 or the parse fails it
    returns -1 and the year stays 0.  Not `featureeng.release_year`, the Spark jobs' rule, which defaults to 1990."""
    if title is None:
        return 0
    t = title.strip(_JAVA_WS)
    if t.isascii():                                # one UTF-16 unit per character
        if len(t) < 6 or not _JAVA_INT.fullmatch(t[-5:-1]):
            return 0
        y = int(t[-5:-1])
        return 0 if y == -1 else y
    u = t.encode("utf-16-le", "surrogatepass")
    n = len(u) // 2
    if n < 6:
        return 0
    try:
        s = u[2 * (n - 5):2 * (n - 1)].decode("utf-16-le")
    except UnicodeDecodeError:                     # half a surrogate pair: not a digit
        return 0
    digits = s[1:] if s[:1] in "+-" else s
    if not digits or not all(c.isdecimal() for c in digits):
        return 0
    y = int("".join(str(int(c)) for c in digits)) * (-1 if s[0] == "-" else 1)
    return 0 if y == -1 else y


def data_manager_titles(path: str) -> List[str]:
    """The title fields (movieData[1], unquoted as Java sees them) of the movies.csv lines DataManager keeps, in the
    order of `data_manager_rows`."""
    titles = []
    with open(path, encoding="utf-8") as f:
        next(f, None)
        for line in f:
            parts = java_split(line.rstrip("\r\n"), ",")
            if len(parts) == 3:
                titles.append(parts[1])
    return titles


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
    there may be at most 64 distinct genres; a violation raises ValueError before any device work.  When `movies` has
    a "title" list, each movie's release year comes from it (`data_manager_release_year`), which multi-channel recall
    needs."""

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
        titles = movies.get("title")
        year = None
        if titles is not None:
            titles = list(titles)
            if len(titles) != ids.shape[0]:
                raise ValueError("movies: %d ids but %d titles" % (ids.shape[0], len(titles)))
            year = np.array([data_manager_release_year(t) for t in titles] or [0], np.int32)
        self.device = device
        self.dim = dim
        self.has_years = year is not None
        lib = _lib.load()
        h = C.c_void_p()
        p = lambda a: a.ctypes.data
        _lib.check(lib.srs_similar_catalog_create_ex_host(p(ids), ids.shape[0], p(off), p(genre), len(vocab),
                                                          p(rmovie), p(rscore), rmovie.shape[0], p(eid), p(emb),
                                                          n_emb, dim, None if year is None else p(year), device,
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

    def _outputs(self, movie_ids, size: int):
        if self._h is None:
            raise ValueError("the catalogue is closed")
        q = np.ascontiguousarray(movie_ids, np.int32).reshape(-1)
        size = int(size)
        if size < 1:
            raise ValueError("size must be >= 1, got %d" % size)
        Q = q.shape[0]
        return q, size, (np.zeros((Q, size), np.int32), np.zeros((Q, size), np.float64), np.zeros(Q, np.int32),
                         np.zeros(Q, np.int32))

    def recommend_arrays(self, movie_ids, size: int, model: str = "emb", candidates: str = "genre"):
        """One device call for every query: (ids int32 [Q, size], scores float64 [Q, size], count int32 [Q],
        status int32 [Q]); row q's first count[q] entries are its list, the rest 0.  `model` "emb" is the cosine
        ranker, any other string calculateSimilarScore, as the Java's switch.  `candidates` "genre" is
        candidateGenerator, "multiple" multipleRetrievalCandidates (which needs the movies' titles)."""
        if candidates not in ("genre", "multiple"):
            raise ValueError("candidates must be 'genre' or 'multiple', got %r" % (candidates,))
        if candidates == "multiple" and not self.has_years:
            raise ValueError("multi-channel recall needs release years: give the movies a 'title' list")
        q, size, out = self._outputs(movie_ids, size)
        m = _lib.SRS_SIMILAR_EMB if model == "emb" else _lib.SRS_SIMILAR_DEFAULT
        p = lambda a: a.ctypes.data
        if candidates == "genre":
            _lib.check(_lib.load().srs_similar_movies_host(self._h, p(q), q.shape[0], size, m, *map(p, out)))
        else:
            _lib.check(_lib.load().srs_similar_movies_candidates_host(
                self._h, _lib.SRS_SIMILAR_CANDIDATES_MULTIPLE, p(q), q.shape[0], size, m, *map(p, out)))
        return out

    def recommend(self, movie_ids, size: int, model: str = "emb", candidates: str = "genre") -> List[SimilarList]:
        """getRecList(movie_id, size, model) for each of `movie_ids`, with the candidates of `candidates`."""
        return _lists(self.recommend_arrays(movie_ids, size, model, candidates))

    def retrieve_by_embedding_arrays(self, movie_ids, size: int):
        """retrievalCandidatesByEmbedding(movie, size) for every query in one device call, laid out as
        `recommend_arrays`: the pool getMovies(10000, "rating"), the query included, by cosine ascending (the
        Java's order: the least similar first, -1 for a movie without a vector, NaN last), ties by movie id."""
        q, size, out = self._outputs(movie_ids, size)
        p = lambda a: a.ctypes.data
        _lib.check(_lib.load().srs_similar_embedding_recall_host(self._h, p(q), q.shape[0], size, *map(p, out)))
        return out

    def retrieve_by_embedding(self, movie_ids, size: int) -> List[SimilarList]:
        """retrievalCandidatesByEmbedding(movie, size) for each of `movie_ids`."""
        return _lists(self.retrieve_by_embedding_arrays(movie_ids, size))


def _lists(arrays) -> List[SimilarList]:
    ids, scores, count, status = arrays
    return [SimilarList(ids[i, :count[i]].copy(), scores[i, :count[i]].copy(), int(status[i]))
            for i in range(ids.shape[0])]


def main(argv: Sequence[str]) -> int:
    import argparse
    ap = argparse.ArgumentParser(prog="python -m sparrowrecsys_b200.similar")
    ap.add_argument("movies")
    ap.add_argument("ratings")
    ap.add_argument("--emb", help="item2vecEmb.csv: id:v v v ... lines")
    ap.add_argument("--model", default="emb", choices=("emb", "default"))
    ap.add_argument("--candidates", default="genre", choices=("genre", "multiple"),
                    help="candidateGenerator (genre) or multipleRetrievalCandidates (multiple)")
    ap.add_argument("--embedding-recall", action="store_true",
                    help="print retrievalCandidatesByEmbedding's list instead of the ranked page (needs --emb)")
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
        movies = {"movieId": movies["movieId"][keep], "genres": [x for x, k in zip(movies["genres"], keep) if k],
                  "title": data_manager_titles(a.movies)}      # the kept lines' fields as Java splits them
    ratings = load_ratings_csv(a.ratings)
    emb = load_embeddings_csv(a.emb) if a.emb else None
    if (a.model == "emb" or a.embedding_recall) and emb is None:
        ap.error("--model emb and --embedding-recall need --emb")
    if a.embedding_recall and a.candidates != "genre":
        ap.error("--embedding-recall is its own candidate source: leave out --candidates")
    queries = movies["movieId"] if a.all else np.array([a.movie], np.int32)
    with SimilarMovies(movies, ratings, emb, a.device) as s:
        lists = (s.retrieve_by_embedding(queries, a.size) if a.embedding_recall
                 else s.recommend(queries, a.size, a.model, a.candidates))
        for mid, r in zip(np.asarray(queries).tolist(), lists):
            if r.status != OK:
                print("%d\t(%s)" % (mid, STATUS_NAMES[r.status]))
            else:
                print("%d\t%s" % (mid, " ".join("%d:%.17g" % (i, x) for i, x in zip(r.movie_ids.tolist(),
                                                                                    r.scores.tolist()))))
    return 0


if __name__ == "__main__":
    import sys
    sys.exit(main(sys.argv[1:]))
