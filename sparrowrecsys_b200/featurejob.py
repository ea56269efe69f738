"""The reference's FeatureEngineering job on the GPU, its Spark ML operators, and the sample / split tail of
FeatureEngForRecModel.

`OFF/featureeng/FeatureEngineering.scala` one-hot encodes movieId, multi-hot encodes the genres (StringIndexer over
the genre words), and turns each movie's rating count, average and variance into a 100-bucket QuantileDiscretizer
bucket and a MinMaxScaler'd average.  `splitAndSaveTrainingTestSamples` (FeatureEngForRecModel.scala:176-188) samples
10 % of the built rows and splits them 0.8 / 0.2; its twin (:190-205) splits at the 0.8 approxQuantile of the
timestamp.  DESIGN.md section 4.16 gives the semantics; `oracle/feature_job.py` restates them in numpy.

* `approx_quantile`, `QuantileDiscretizer(...).fit(x)` -> `Bucketizer`, `MinMaxScaler`, `StringIndexer`: the
  operators, each a device call (`srs_*_host` in include/srs_ctr.h).
* `rating_features`, `one_hot`, `multi_hot` and `feature_engineering(ratings, movies)`: the job's three results.
* `split_samples` / `split_samples_by_timestamp`: `build_samples` output -> training and test feature dicts, in
  its keys and dtypes, so they go straight into `write_samples_csv`, `predict`, `evaluate` and `Trainer.fit`.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Mapping, Sequence, Tuple

import numpy as np

from . import _lib

_M64 = (1 << 64) - 1


def _p(a):
    return a.ctypes.data


def _values(x) -> np.ndarray:
    v = np.ascontiguousarray(x, np.float64).reshape(-1)
    if v.size == 0:
        raise ValueError("no values")
    return v


def approx_quantile(values, probabilities: Sequence[float], relative_error: float, device: int = 0) -> np.ndarray:
    """Dataset.stat.approxQuantile(col, probabilities, relative_error) as Spark 2.4.3's QuantileSummaries answers it
    with every value in one summary (float64 per probability).  NaN values raise ValueError."""
    v = _values(values)
    p = np.ascontiguousarray(probabilities, np.float64).reshape(-1)
    out = np.zeros(max(p.size, 1), np.float64)
    _lib.check(_lib.load().srs_approx_quantile_host(_p(v), v.size, _p(p), p.size, float(relative_error), device,
                                                    _p(out)))
    return out[:p.size]


class Bucketizer:
    """Bucketizer(splits), handleInvalid "error": bucket k holds [splits[k], splits[k + 1]), the last one includes
    its upper split.  `transform` returns float64 bucket ids, as Spark's output column."""

    def __init__(self, splits):
        self.splits = np.ascontiguousarray(splits, np.float64).reshape(-1)

    def transform(self, values, device: int = 0) -> np.ndarray:
        v = _values(values)
        out = np.zeros(v.size, np.int32)
        _lib.check(_lib.load().srs_bucketize_host(_p(self.splits), self.splits.size, _p(v), v.size, device, _p(out)))
        return out.astype(np.float64)


class QuantileDiscretizer:
    """QuantileDiscretizer(numBuckets, relativeError): `fit` gives the Bucketizer whose splits are the
    approxQuantile at k / numBuckets, ends replaced by -inf / +inf, duplicates removed (so equal values can leave
    fewer buckets)."""

    def __init__(self, num_buckets: int = 2, relative_error: float = 0.001):
        self.num_buckets, self.relative_error = int(num_buckets), float(relative_error)

    def _run(self, values, device, with_buckets):
        v = _values(values)
        splits = np.zeros(max(self.num_buckets, 1) + 1, np.float64)
        ns = C.c_int32(0)
        b = np.zeros(v.size, np.int32)
        _lib.check(_lib.load().srs_quantile_discretizer_host(_p(v), v.size, self.num_buckets, self.relative_error,
                                                             device, _p(splits), C.byref(ns),
                                                             _p(b) if with_buckets else None))
        return Bucketizer(splits[:ns.value].copy()), b.astype(np.float64)

    def fit(self, values, device: int = 0) -> Bucketizer:
        return self._run(values, device, False)[0]

    def fit_transform(self, values, device: int = 0) -> Tuple[Bucketizer, np.ndarray]:
        """fit(values) and its transform of the same values, in one device call."""
        return self._run(values, device, True)


class MinMaxScalerModel:
    def __init__(self, original_min: float, original_max: float):
        self.original_min, self.original_max = float(original_min), float(original_max)

    def transform(self, values, device: int = 0) -> np.ndarray:
        """(x - Emin) / (Emax - Emin), 0.5 when Emax == Emin (float64)."""
        return _minmax(values, np.array([self.original_min, self.original_max]), device)[0]


def _minmax(values, fit, device):
    v = _values(values)
    out = np.zeros(v.size, np.float64)
    mm = np.zeros(2, np.float64)
    _lib.check(_lib.load().srs_minmax_scale_host(_p(v), v.size, None if fit is None else _p(fit), device, _p(out),
                                                 _p(mm)))
    return out, mm


class MinMaxScaler:
    """MinMaxScaler with Spark's defaults (min 0, max 1) over one column."""

    def fit(self, values, device: int = 0) -> MinMaxScalerModel:
        return MinMaxScalerModel(*_minmax(values, None, device)[1])

    def fit_transform(self, values, device: int = 0) -> Tuple[MinMaxScalerModel, np.ndarray]:
        out, mm = _minmax(values, None, device)
        return MinMaxScalerModel(*mm), out


def _word_ids(tokens: Sequence[str]):
    from .featureeng import java_string_hash
    ids: Dict[str, int] = {}
    tok = np.array([ids.setdefault(t, len(ids)) for t in tokens], np.int32)
    words = list(ids)
    return tok, words, np.array([java_string_hash(w) for w in words], np.int32)


class StringIndexerModel:
    def __init__(self, labels: Sequence[str], counts: Sequence[int]):
        self.labels, self.counts = list(labels), list(counts)
        self._index = {w: k for k, w in enumerate(self.labels)}

    def transform(self, values: Sequence[str]) -> np.ndarray:
        """The label index of each value (float64); an unseen label raises KeyError (handleInvalid "error")."""
        return np.array([self._index[v] for v in values], np.float64)


class StringIndexer:
    """StringIndexer (stringOrderType frequencyDesc): labels by descending count, ties in the iteration order of
    the Scala 2.11 immutable.HashMap that countByValue builds."""

    def fit(self, values: Sequence[str], device: int = 0) -> StringIndexerModel:
        tok, words, hashes = _word_ids(list(values))
        if tok.size == 0:
            raise ValueError("no values")
        lw = np.zeros(len(words), np.int32)
        lc = np.zeros(len(words), np.int64)
        _lib.check(_lib.load().srs_string_indexer_host(_p(tok), tok.size, _p(hashes), len(words), device, _p(lw),
                                                       _p(lc)))
        return StringIndexerModel([words[w] for w in lw.tolist()], lc.tolist())


def one_hot(movie_ids) -> Dict[str, object]:
    """oneHotEncoderExample: OneHotEncoderEstimator(dropLast = false) on movieId cast to int.  Per row (input order)
    the index of its one 1.0, and the vector size max + 1."""
    ids = np.asarray(movie_ids, np.int64)
    if ids.size == 0 or ids.min() < 0 or ids.max() >= 2 ** 31 - 1:
        raise ValueError("movie ids must be non-empty and in 0..2^31 - 2")
    return {"movieIdNumber": ids.astype(np.int32), "index": ids.astype(np.int32), "size": int(ids.max()) + 1}


def multi_hot(movie_ids, genres: Sequence[str], device: int = 0) -> Dict[str, object]:
    """multiHotEncoderExample: StringIndexer over the `|`-separated genre words of every movie, then per movie,
    ascending id, a sparse vector of size = the number of labels whose indices are its words' labels, sorted.
    Returns labels, counts, movieId, CSR offsets / indices (int32) and size.  A movie listing one genre twice, or
    a movie id given twice, raises ValueError."""
    ids = np.ascontiguousarray(movie_ids, np.int32)
    lists = [g.split("|") for g in genres]
    if len(lists) != ids.size or ids.size == 0:
        raise ValueError("movie ids and genres differ in length, or are empty")
    tok, words, hashes = _word_ids([w for gl in lists for w in gl])
    off = np.zeros(ids.size + 1, np.int32)
    np.cumsum([len(gl) for gl in lists], out=off[1:])
    W = len(words)
    lw, lc = np.zeros(W, np.int32), np.zeros(W, np.int64)
    om, oo, oi = np.zeros(ids.size, np.int32), np.zeros(ids.size + 1, np.int32), np.zeros(tok.size, np.int32)
    _lib.check(_lib.load().srs_genre_multihot_host(_p(ids), _p(off), _p(tok), ids.size, _p(hashes), W, device,
                                                   _p(lw), _p(lc), _p(om), _p(oo), _p(oi)))
    return {"labels": [words[w] for w in lw.tolist()], "counts": lc, "movieId": om, "offsets": oo, "indices": oi,
            "size": W}


def _half_stars(ratings: Mapping[str, np.ndarray]):
    movie = np.ascontiguousarray(ratings["movieId"], np.int32)
    r2 = np.asarray(ratings["rating"], np.float64) * 2
    if r2.shape != movie.shape:
        raise ValueError("ratings columns differ in length")
    if not np.array_equal(r2, np.trunc(r2)) or (r2.size and (r2.min() < 1 or r2.max() > 10)):
        raise ValueError("ratings must be half-stars in [0.5, 5]")
    return movie, np.ascontiguousarray(r2, np.int8)


def rating_features(ratings: Mapping[str, np.ndarray], device: int = 0) -> Dict[str, np.ndarray]:
    """ratingFeatures' groupBy(movieId): movieId (int32, ascending), ratingCount (int64), avgRating and ratingVar
    (float64; var_samp, NaN for the null of a one-rating movie), each the correctly rounded value of exact sums."""
    movie, half = _half_stars(ratings)
    cap = int(movie.max(initial=0)) + 1
    ids, cnt = np.zeros(cap, np.int32), np.zeros(cap, np.int64)
    avg, var = np.zeros(cap, np.float64), np.zeros(cap, np.float64)
    m = C.c_int32(0)
    _lib.check(_lib.load().srs_rating_features_host(_p(movie), _p(half), movie.size, device, cap, _p(ids), _p(cnt),
                                                    _p(avg), _p(var), C.byref(m)))
    k = m.value
    return {"movieId": ids[:k], "ratingCount": cnt[:k], "avgRating": avg[:k], "ratingVar": var[:k]}


def feature_engineering(ratings: Mapping[str, np.ndarray], movies: Mapping[str, object], device: int = 0,
                        num_buckets: int = 100, relative_error: float = 0.001) -> Dict[str, Dict[str, object]]:
    """The whole FeatureEngineering job: "one_hot" and "multi_hot" of movies.csv (`one_hot`, `multi_hot`), and
    "movie_features", the ratingFeatures pipeline - `rating_features`, then QuantileDiscretizer(num_buckets) on
    ratingCount -> ratingCountBucket and MinMaxScaler on avgRating -> scaleAvgRating; its "splits" are the
    discretizer's."""
    mf = rating_features(ratings, device)
    bucketizer, buckets = QuantileDiscretizer(num_buckets, relative_error).fit_transform(
        mf["ratingCount"].astype(np.float64), device)
    mf["ratingCountBucket"] = buckets
    mf["scaleAvgRating"] = MinMaxScaler().fit_transform(mf["avgRating"], device)[1]
    mf["splits"] = bucketizer.splits
    return {"one_hot": one_hot(movies["movieId"]), "multi_hot": multi_hot(movies["movieId"], movies["genres"], device),
            "movie_features": mf}


# ------------------------------------------------------------------------------------------------ sample, split
def sample_split_rows(n: int, seed: int, fraction: float = 0.1, weights: Sequence[float] = (0.8, 0.2),
                      device: int = 0) -> List[np.ndarray]:
    """The row indices (int64, ascending) of each part of sample(fraction).randomSplit(weights) over n rows."""
    w = np.ascontiguousarray(weights, np.float64).reshape(-1)
    rows = np.zeros(max(int(n), 1), np.int32)
    cnt = np.zeros(max(w.size, 1), np.int64)
    _lib.check(_lib.load().srs_sample_split_host(int(n), int(seed) & _M64, float(fraction), _p(w), w.size, device,
                                                 _p(rows), _p(cnt)))
    ends = np.cumsum(cnt[:w.size])
    return [rows[e - c:e].astype(np.int64) for c, e in zip(cnt[:w.size], ends)]


def sample_split_rows_by_timestamp(timestamp, seed: int, fraction: float = 0.1, relative_error: float = 0.05,
                                   device: int = 0) -> Tuple[np.ndarray, np.ndarray, float]:
    """(training rows, test rows, split timestamp) of sample(fraction) split at approxQuantile(timestamp, 0.8):
    sampled rows with timestamp <= the split train.  The split is NaN when no row is sampled."""
    ts = np.ascontiguousarray(timestamp, np.int64).reshape(-1)
    rows = np.zeros(max(ts.size, 1), np.int32)
    cnt = np.zeros(2, np.int64)
    split = C.c_double(0.0)
    _lib.check(_lib.load().srs_sample_split_by_timestamp_host(_p(ts), ts.size, int(seed) & _M64, float(fraction),
                                                              float(relative_error), device, _p(rows), _p(cnt),
                                                              C.byref(split)))
    a, b = int(cnt[0]), int(cnt[1])
    return rows[:a].astype(np.int64), rows[a:a + b].astype(np.int64), split.value


def _take(samples: Mapping[str, np.ndarray], rows: np.ndarray) -> Dict[str, np.ndarray]:
    return {k: np.asarray(v)[rows] for k, v in samples.items()}


def split_samples(samples: Mapping[str, np.ndarray], seed: int, fraction: float = 0.1,
                  weights: Sequence[float] = (0.8, 0.2), device: int = 0) -> List[Dict[str, np.ndarray]]:
    """splitAndSaveTrainingTestSamples: sample(fraction), then randomSplit(weights), on counter-based uniforms keyed
    by `seed` (the sample and the split draw from two streams, so the weights do not change which rows are
    sampled).  One feature dict per weight, rows in input order, keys and dtypes as `samples`."""
    n = len(next(iter(samples.values())))
    return [_take(samples, r) for r in sample_split_rows(n, seed, fraction, weights, device)]


def split_samples_by_timestamp(samples: Mapping[str, np.ndarray], seed: int, fraction: float = 0.1,
                               relative_error: float = 0.05, device: int = 0
                               ) -> Tuple[Dict[str, np.ndarray], Dict[str, np.ndarray]]:
    """splitAndSaveTrainingTestSamplesByTimeStamp: the same sample, then the rows with timestamp <= the sample's
    approxQuantile(timestamp, 0.8, relative_error) train and the rest test.  (training, test) feature dicts, rows
    in input order."""
    tr, te, _ = sample_split_rows_by_timestamp(samples["timestamp"], seed, fraction, relative_error, device)
    return _take(samples, tr), _take(samples, te)
