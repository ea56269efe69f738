"""Build the CTR training samples from ratings.csv + movies.csv on the GPU.

This is the reference's Spark job `FeatureEngForRecModel.scala:21-130`: each rating becomes one 27-column sample
row (label, movie features over all ratings of the movie, user features over the user's previous 100 ratings),
rows with fewer than two earlier ratings of the user dropped.  DESIGN.md section 4.11 gives the semantics and the
order rules; `oracle/feature_eng.py` restates them in numpy.

* `load_ratings_csv` / `load_movies_csv` read the reference's CSVs; the title -> release-year rule runs here on the
  host (`release_year`).
* `build_samples` runs the job on one device (`srs_featureeng_host`) and returns the rows in ratings.csv order,
  keyed and typed exactly as `features.load_samples_csv` returns them, so the result goes straight into
  `predict`, `evaluate` and `Trainer.fit`.
* `write_samples_csv` writes rows in the reference's text format.
* `feature_engineering`, `split_samples` and `split_samples_by_timestamp` (from `featurejob`, DESIGN.md section
  4.16) run the FeatureEngineering job and the sample / split that turns these rows into trainingSamples.csv and
  testSamples.csv.

    python -m sparrowrecsys_b200.featureeng samples RATINGS MOVIES OUT.csv
    python -m sparrowrecsys_b200.featureeng job RATINGS MOVIES
    python -m sparrowrecsys_b200.featureeng split RATINGS MOVIES OUT_DIR [--by-timestamp] [--seed S]
"""
from __future__ import annotations

import csv
import ctypes as C
import re
from typing import Dict, List, Mapping, Sequence

import numpy as np

from . import _lib
from .featurejob import feature_engineering, split_samples, split_samples_by_timestamp  # noqa: F401

DEFAULT_YEAR = 1990
MAX_GENRE_WORDS = 24

COLUMNS = ("movieId", "userId", "rating", "timestamp", "label", "releaseYear", "movieGenre1", "movieGenre2",
           "movieGenre3", "movieRatingCount", "movieAvgRating", "movieRatingStddev", "userRatedMovie1",
           "userRatedMovie2", "userRatedMovie3", "userRatedMovie4", "userRatedMovie5", "userRatingCount",
           "userAvgReleaseYear", "userReleaseYearStddev", "userAvgRating", "userRatingStddev", "userGenre1",
           "userGenre2", "userGenre3", "userGenre4", "userGenre5")
_TWO_DECIMALS = ("movieAvgRating", "movieRatingStddev", "userReleaseYearStddev", "userAvgRating", "userRatingStddev")
_GENRE_COLS = ("movieGenre1", "movieGenre2", "movieGenre3", "userGenre1", "userGenre2", "userGenre3", "userGenre4",
               "userGenre5")

_JAVA_WS = "".join(chr(c) for c in range(33))          # java.lang.String.trim strips every char <= ' '
_JAVA_INT = re.compile(r"[+-]?[0-9]+\Z")


def release_year(title) -> int:
    """The reference's title UDF: `title.trim.substring(title.length - 5, title.length - 1).toInt` - the substring
    bounds use the *untrimmed* length - and 1990 for a missing title or a trimmed title shorter than 6 characters.
    Where the reference would throw (bounds past the trimmed title, or not an integer) this raises ValueError."""
    if title is None:
        return DEFAULT_YEAR
    t = title.strip(_JAVA_WS)
    if len(t) < 6:
        return DEFAULT_YEAR
    if len(title) - 1 > len(t):
        raise ValueError("title %r: its year substring ends past the trimmed title" % (title,))
    s = t[len(title) - 5:len(title) - 1]
    if not _JAVA_INT.match(s):
        raise ValueError("title %r: %r is not an integer" % (title, s))
    return int(s)


def java_string_hash(s: str) -> int:
    """java.lang.String.hashCode (UTF-16 code units), as a signed 32-bit int."""
    b = s.encode("utf-16-le")
    h = 0
    for i in range(0, len(b), 2):
        h = (31 * h + (b[i] | (b[i + 1] << 8))) & 0xFFFFFFFF
    return h - (1 << 32) if h >= 1 << 31 else h


def load_ratings_csv(path: str) -> Dict[str, np.ndarray]:
    """ratings.csv (userId,movieId,rating,timestamp) in file order: ids and timestamp int32, rating float64."""
    a = np.loadtxt(path, delimiter=",", skiprows=1, dtype=np.float64, ndmin=2)
    if a.shape[0] and a.shape[1] != 4:
        raise ValueError("%s: expected 4 columns, got %d" % (path, a.shape[1]))
    a = a.reshape(-1, 4)
    out = {"rating": a[:, 2].copy()}
    for j, k in ((0, "userId"), (1, "movieId"), (3, "timestamp")):
        v = a[:, j]
        if not np.array_equal(v, np.trunc(v)) or (v.size and (v.min() < -2 ** 31 or v.max() >= 2 ** 31)):
            raise ValueError("%s: column %s is not int32" % (path, k))
        out[k] = v.astype(np.int32)
    return out


def load_movies_csv(path: str) -> Dict[str, object]:
    """movies.csv (movieId,title,genres): movieId int32, title and genres as lists of str, and releaseYear int32
    from the title rule (`release_year`)."""
    with open(path, newline="", encoding="utf-8") as f:
        rows = list(csv.reader(f))[1:]
    title = [r[1] for r in rows]
    return {"movieId": np.array([int(r[0]) for r in rows], np.int32), "title": title,
            "genres": [r[2] for r in rows], "releaseYear": np.array([release_year(t) for t in title], np.int32)}


def _movie_table(movies: Mapping[str, object], n_slots: int):
    words: Dict[str, int] = {}
    lists = [[words.setdefault(w, len(words)) for w in g.split("|")] for g in movies["genres"]]
    if len(words) > MAX_GENRE_WORDS:
        raise ValueError("%d distinct genre words; at most %d are supported" % (len(words), MAX_GENRE_WORDS))
    L = max([len(x) for x in lists] + [3])
    if L > MAX_GENRE_WORDS:
        raise ValueError("a movie lists %d genres; at most %d are supported" % (L, MAX_GENRE_WORDS))
    years = movies.get("releaseYear")
    if years is None:
        years = [release_year(t) for t in movies["title"]]
    year = np.full(n_slots, DEFAULT_YEAR, np.int32)
    genres = np.full((n_slots, L), -1, np.int32)
    for mid, y, gl in zip(np.asarray(movies["movieId"]).tolist(), np.asarray(years).tolist(), lists):
        year[mid] = y
        genres[mid, :len(gl)] = gl
    return year, genres, list(words)


def build_samples(ratings: Mapping[str, np.ndarray], movies: Mapping[str, object], device: int = 0
                  ) -> Dict[str, np.ndarray]:
    """The sample rows of `ratings` (userId, movieId, rating, timestamp; as `load_ratings_csv` returns) and `movies`
    (movieId, title, genres, optionally releaseYear; as `load_movies_csv` returns), built on `device`.  Rows are in
    ratings order; keys and dtypes are those of `features.load_samples_csv` (genres as str, "" for none; a missing
    userRatedMovie is 0).  Ids must be >= 0 and ratings half-stars in [0.5, 5]: a violation raises ValueError
    before any device work."""
    user = np.ascontiguousarray(ratings["userId"], np.int32)
    movie = np.ascontiguousarray(ratings["movieId"], np.int32)
    ts = np.ascontiguousarray(ratings["timestamp"], np.int32)
    r2 = np.asarray(ratings["rating"], np.float64) * 2
    n = user.shape[0]
    if movie.shape[0] != n or ts.shape[0] != n or r2.shape[0] != n:
        raise ValueError("ratings columns differ in length")
    if not np.array_equal(r2, np.trunc(r2)) or (n and (r2.min() < 1 or r2.max() > 10)):
        raise ValueError("ratings must be half-stars in [0.5, 5]")
    half = np.ascontiguousarray(r2, np.int8)
    mids = np.asarray(movies["movieId"])
    if (mids.size and mids.min() < 0) or (n and movie.min() < 0):
        raise ValueError("negative movie id")
    n_slots = int(max(movie.max(initial=0), mids.max(initial=0))) + 1
    year, genres, words = _movie_table(movies, n_slots)
    hashes = np.array([java_string_hash(w) for w in words] or [0], np.int32)

    cap = max(n, 1)
    i32 = lambda *shape: np.zeros((cap,) + shape, np.int32)
    f32 = lambda: np.zeros(cap, np.float32)
    o = {"row": i32(), "label": i32(), "release_year": i32(), "movie_genre": i32(3), "movie_rating_count": i32(),
         "movie_avg_rating": f32(), "movie_rating_stddev": f32(), "user_rated_movie": i32(5),
         "user_rating_count": i32(), "user_avg_release_year": f32(), "user_release_year_stddev": f32(),
         "user_avg_rating": f32(), "user_rating_stddev": f32(), "user_genre": i32(5)}
    st = _lib.SrsSamples(**{k: v.ctypes.data for k, v in o.items()})
    kept = C.c_int64(0)
    lib = _lib.load()
    p = lambda a: a.ctypes.data
    _lib.check(lib.srs_featureeng_host(p(user), p(movie), p(half), p(ts), n, p(year), p(genres), n_slots,
                                       genres.shape[1], p(hashes), len(words), device, C.byref(st), C.byref(kept)))
    k = kept.value
    o = {key: v[:k] for key, v in o.items()}
    rows = o["row"]
    word = np.array(words + [""], dtype=object)
    name = lambda idx: word[np.where(idx >= 0, idx, len(words))]
    out = {"movieId": movie[rows], "userId": user[rows], "rating": (half[rows] / np.float32(2)).astype(np.float32),
           "timestamp": ts[rows], "label": o["label"], "releaseYear": o["release_year"],
           "movieRatingCount": o["movie_rating_count"], "movieAvgRating": o["movie_avg_rating"],
           "movieRatingStddev": o["movie_rating_stddev"], "userRatingCount": o["user_rating_count"],
           "userAvgReleaseYear": o["user_avg_release_year"], "userReleaseYearStddev": o["user_release_year_stddev"],
           "userAvgRating": o["user_avg_rating"], "userRatingStddev": o["user_rating_stddev"]}
    for j in range(3):
        out["movieGenre%d" % (j + 1)] = name(o["movie_genre"][:, j])
    for j in range(5):
        out["userRatedMovie%d" % (j + 1)] = np.ascontiguousarray(o["user_rated_movie"][:, j])
        out["userGenre%d" % (j + 1)] = name(o["user_genre"][:, j])
    return {c: out[c] for c in COLUMNS}


def _text(v: str) -> str:
    return '""' if v == "" else ('"%s"' % v if "," in v else v)


def write_samples_csv(path: str, samples: Mapping[str, Sequence]) -> None:
    """Write sample rows in the reference's text format (modelSamples.csv): the 27 columns in its header order,
    ratings with one decimal, two-decimal columns as java.text.DecimalFormat "#,##0.00" prints them (a grouping
    comma from 1 000 up; no column of MovieLens data reaches it), `""` for an empty genre and for a userRatedMovie of
    0 (MovieLens ids start at 1; `load_samples_csv` reads both as 0)."""
    cols: List[List[str]] = []
    for c in COLUMNS:
        v = samples[c]
        if c in _GENRE_COLS:
            cols.append([_text(str(x)) for x in v])
        elif c == "rating":
            cols.append(["%.1f" % x for x in np.asarray(v, np.float64)])
        elif c in _TWO_DECIMALS:
            cols.append([_text("{:,.2f}".format(x)) for x in np.asarray(v, np.float64)])
        elif c.startswith("userRatedMovie"):
            cols.append(['""' if x == 0 else str(x) for x in np.asarray(v).astype(np.int64).tolist()])
        else:
            cols.append([str(x) for x in np.asarray(v).astype(np.int64).tolist()])
    with open(path, "w", newline="") as f:
        f.write(",".join(COLUMNS) + "\n")
        for row in zip(*cols):
            f.write(",".join(row) + "\n")


def _show(title: str, cols: Mapping[str, Sequence], rows: int = 10) -> None:
    names = list(cols)
    print(title)
    print("|".join(names))
    for i in range(min(rows, len(cols[names[0]]))):
        print("|".join(str(cols[c][i]) for c in names))
    print()


def main(argv: Sequence[str]) -> int:
    """`samples`: build_samples -> OUT.csv; `job`: the FeatureEngineering job, printing the first 10 rows of each
    result as its show(10) calls do; `split`: build the samples, sample 10 % and write OUT_DIR/trainingSamples.csv
    and OUT_DIR/testSamples.csv (0.8 / 0.2 at random, or at the 0.8 timestamp quantile with --by-timestamp)."""
    import argparse
    import os
    ap = argparse.ArgumentParser(prog="python -m sparrowrecsys_b200.featureeng")
    ap.add_argument("mode", choices=("samples", "job", "split"))
    ap.add_argument("ratings")
    ap.add_argument("movies")
    ap.add_argument("out", nargs="?")
    ap.add_argument("--by-timestamp", action="store_true")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    ratings, movies = load_ratings_csv(a.ratings), load_movies_csv(a.movies)
    if a.mode == "job":
        r = feature_engineering(ratings, movies, a.device)
        oh, mh, mf = r["one_hot"], r["multi_hot"], r["movie_features"]
        _show("OneHotEncoder Example:", {"movieId": movies["movieId"], "movieIdVector": [
            "(%d,[%d],[1.0])" % (oh["size"], i) for i in oh["index"][:10]]})
        vec = ["(%d,[%s],[%s])" % (mh["size"], ",".join(map(str, mh["indices"][b:e])), ",".join(["1.0"] * (e - b)))
               for b, e in zip(mh["offsets"][:10], mh["offsets"][1:11])]
        _show("MultiHotEncoder Example:", {"movieId": mh["movieId"], "vector": vec})
        _show("Numerical features Example:", {k: mf[k] for k in ("movieId", "ratingCount", "avgRating", "ratingVar",
                                                                 "ratingCountBucket", "scaleAvgRating")})
        return 0
    if not a.out:
        ap.error("%s needs an output path" % a.mode)
    samples = build_samples(ratings, movies, a.device)
    if a.mode == "samples":
        write_samples_csv(a.out, samples)
        return 0
    if a.by_timestamp:
        train, test = split_samples_by_timestamp(samples, a.seed, device=a.device)
    else:
        train, test = split_samples(samples, a.seed, device=a.device)
    os.makedirs(a.out, exist_ok=True)
    write_samples_csv(os.path.join(a.out, "trainingSamples.csv"), train)
    write_samples_csv(os.path.join(a.out, "testSamples.csv"), test)
    print("%d training and %d test rows in %s" % (len(train["movieId"]), len(test["movieId"]), a.out))
    return 0


if __name__ == "__main__":
    import sys
    sys.exit(main(sys.argv[1:]))
