"""Host-side feature handling for the CTR forward path.

Two jobs, both host logic that sits *above* the C-ABI:

* `load_samples_csv` reproduces what the reference's `get_dataset`
  (`TFRecModel/.../DIN.py:14-22`: `make_csv_dataset(..., na_value="0")`) hands to
  `model.predict`, minus batching and shuffling: a dict of 1-D column arrays keyed
  by the CSV header, ids/counts as int32, ratings as float32, genres as `str`,
  empty int -> 0, empty float -> 0.0, empty string -> "".
* `encode_batch` turns such a feature dict (the argument of `predict`) into the
  flat integer / float arrays the C-ABI takes: the genre vocabulary lookup that
  TF does with a `LookupTableFindV2` op inside the graph is done here with a
  dict (OOV / "" -> -1, SURVEY.md section 8a item 3); the kernels only ever see
  int32 ids and float32 numerics.
"""
from __future__ import annotations

import csv
from typing import Dict, Mapping, Optional, Sequence

import numpy as np

from .spec import (GENRE_VOCAB, MOVIE_GENRE_KEYS, NUMERIC_KEYS, USER_GENRE_KEYS,
                   ModelSpec, history_keys)

_GENRE_INDEX = {g: i for i, g in enumerate(GENRE_VOCAB)}
_GENRE_LOOKUP = {**_GENRE_INDEX, **{g.encode(): i for g, i in _GENRE_INDEX.items()}}   # str and bytes keys

_FLOAT_COLS = {"rating", "movieAvgRating", "movieRatingStddev", "userAvgRating",
               "userRatingStddev", "userReleaseYearStddev"}
_STRING_COLS = set(MOVIE_GENRE_KEYS) | set(USER_GENRE_KEYS)


def load_samples_csv(path: str, max_rows: Optional[int] = None) -> Dict[str, np.ndarray]:
    """Read a SparrowRecSys sample CSV in file order (no shuffle).

    Column typing follows what `make_csv_dataset` infers on the bundled files
    (SURVEY.md section 8a front matter); `userAvgReleaseYear` is integer-valued in the
    bundled data but is parsed as float to be safe (no model reads it).
    """
    with open(path, newline="") as f:
        reader = csv.reader(f)
        header = next(reader)
        cols = [[] for _ in header]
        for n, row in enumerate(reader):
            if max_rows is not None and n >= max_rows:
                break
            if len(row) != len(header):     # ignore_errors=True drops malformed lines
                continue
            for c, v in zip(cols, row):
                c.append(v)
    out: Dict[str, np.ndarray] = {}
    for name, vals in zip(header, cols):
        if name in _STRING_COLS:
            out[name] = np.array(vals, dtype=object)
        elif name in _FLOAT_COLS or name == "userAvgReleaseYear":
            out[name] = np.array([float(v) if v != "" else 0.0 for v in vals], dtype=np.float32)
        else:
            out[name] = np.array([int(v) if v != "" else 0 for v in vals], dtype=np.int32)
    return out


def genre_to_index(values) -> np.ndarray:
    """Vocabulary lookup of `categorical_column_with_vocabulary_list` (default
    `default_value=-1`, `num_oov_buckets=0`): known genre (str or bytes) -> position, else -1."""
    arr = np.asarray(values)
    if arr.dtype.kind in "iu":          # already indexed by the caller
        return arr.astype(np.int32)
    flat = arr.ravel()
    get = _GENRE_LOOKUP.get             # one dict probe per element (~0.1 us)
    return np.fromiter((get(v, -1) for v in flat.tolist()), np.int32, count=flat.shape[0]).reshape(arr.shape)


def _as_1d(features: Mapping[str, object], key: str) -> np.ndarray:
    if key not in features:
        raise KeyError("missing required feature %r" % key)
    a = np.asarray(features[key])
    if a.ndim == 2 and a.shape[1] == 1:
        a = a[:, 0]
    if a.ndim != 1:
        raise ValueError("feature %r must be 1-D [B], got shape %s" % (key, a.shape))
    return a


def _as_ids(features, key, limit, what) -> np.ndarray:
    a = _as_1d(features, key)
    if a.dtype.kind == "f":
        a = a.astype(np.int64)
    a64 = a.astype(np.int64)
    if a64.size and (a64.min() < 0 or a64.max() >= limit):
        # categorical_column_with_identity asserts 0 <= id < num_buckets
        # (assert_greater_or_equal_0 / assert_less_than_num_buckets in the shipped
        # saved_model.pb; SURVEY.md section 8a item 4)
        raise ValueError("%s %r out of range [0, %d)" % (what, key, limit))
    return a64.astype(np.int32)


class EncodedBatch:
    """Flat arrays for one batch, in the layout of `srs_batch` (include/srs_ctr.h)."""
    __slots__ = ("B", "movie_id", "user_id", "hist", "movie_genre", "user_genre", "numerics")

    def __init__(self, B, movie_id, user_id, hist, movie_genre, user_genre, numerics):
        self.B = B
        self.movie_id = movie_id        # int32 [B]
        self.user_id = user_id          # int32 [B]
        self.hist = hist                # int32 [B, T] (uint16 with narrow_ids) or None
        self.movie_genre = movie_genre  # int32 [B, 3] (-1 = missing/OOV) or None
        self.user_genre = user_genre    # int32 [B, 5] or None
        self.numerics = numerics        # float32 [B, 7] in NUMERIC_KEYS order or None

    def slice(self, lo: int, hi: int) -> "EncodedBatch":
        s = lambda a: None if a is None else a[lo:hi]
        return EncodedBatch(hi - lo, s(self.movie_id), s(self.user_id), s(self.hist),
                            s(self.movie_genre), s(self.user_genre), s(self.numerics))


def encode_batch(spec: ModelSpec, features: Mapping[str, object], arena_alloc=None,
                 narrow_ids: bool = False) -> EncodedBatch:
    """Feature dict (keys as in the Keras `inputs` dicts, e.g. DIN.py:34-59) ->
    `EncodedBatch`.  Unknown keys are ignored (the reference datasets carry
    `rating`, `timestamp`, ... which no model reads); a missing required key raises
    `KeyError`; an out-of-range id raises `ValueError`.  `arena_alloc(nbytes)` may supply
    the backing uint8 buffer (e.g. pinned memory); the arrays are views into it, back to
    back in the packed order the library recognises.  `narrow_ids`: store the history ids as
    uint16 (`srs_batch::hist16`; vocabularies of at most 65536 movies) - the history is most
    of a DIN batch, so the host-to-device copy roughly halves."""
    m = spec.model
    movie_id_in = _as_ids(features, "movieId", spec.n_movies, "movie id")
    user_id_in = _as_ids(features, "userId", spec.n_users, "user id")
    B = movie_id_in.shape[0]
    if user_id_in.shape[0] != B:
        raise ValueError("userId and movieId differ in length")
    hist = movie_genre = user_genre = numerics = None
    # one arena in the packed order of include/srs_ctr.h (srs_batch): the library then moves
    # the whole batch host->device with a single copy
    hist_keys = history_keys(spec.hist_len) if m in ("din", "dien") \
        else (["userRatedMovie1"] if m == "widendeep" else [])
    dense = m not in ("neuralcf", "twotowers")
    narrow = bool(narrow_ids) and bool(hist_keys)
    if narrow and spec.n_movies > 65536:
        raise ValueError("narrow_ids needs a movie vocabulary of at most 65536 ids")
    hist_bytes = (B * len(hist_keys) * 2 + 3) & ~3 if narrow else B * len(hist_keys) * 4
    nbytes = B * (2 + (15 if dense else 0)) * 4 + hist_bytes
    arena = arena_alloc(nbytes) if arena_alloc is not None else np.empty(nbytes, np.uint8)
    cursor = [0]

    def carve(shape, dtype):
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        view = arena[cursor[0]:cursor[0] + n].view(dtype).reshape(shape)
        cursor[0] += (n + 3) & ~3
        return view

    movie_id = carve((B,), np.int32)
    movie_id[:] = movie_id_in
    user_id = carve((B,), np.int32)
    user_id[:] = user_id_in
    if hist_keys:
        hist = carve((B, len(hist_keys)), np.uint16 if narrow else np.int32)
        for p, k in enumerate(hist_keys):
            hist[:, p] = _as_ids(features, k, spec.n_movies, "history movie id")
    if dense:
        movie_genre = carve((B, 3), np.int32)
        user_genre = carve((B, 5), np.int32)
        numerics = carve((B, len(NUMERIC_KEYS)), np.float32)
        movie_genre[:] = -1
        user_genre[:] = -1
        for j, k in enumerate(NUMERIC_KEYS):
            numerics[:, j] = _as_1d(features, k).astype(np.float32)   # numeric_column casts
        n_mg = 3 if m in ("embeddingmlp", "widendeep") else 1
        n_ug = 5 if m in ("embeddingmlp", "widendeep") else 1
        for j in range(n_mg):
            movie_genre[:, j] = genre_to_index(_as_1d(features, MOVIE_GENRE_KEYS[j]))
        for j in range(n_ug):
            user_genre[:, j] = genre_to_index(_as_1d(features, USER_GENRE_KEYS[j]))
        if (movie_genre >= spec.n_genres).any() or (user_genre >= spec.n_genres).any():
            raise ValueError("genre index out of vocabulary range")
    for a in (hist, movie_genre, user_genre, numerics):
        if a is not None and a.shape[0] != B:
            raise ValueError("feature columns differ in length")
    return EncodedBatch(B, movie_id, user_id, hist, movie_genre, user_genre, numerics)


def negative_history_keys(T: int):
    """The DIEN negative-sample inputs `negtive_userRatedMovie2..T` (sic, DIEN.py:83-86), graph order."""
    return ["negtive_userRatedMovie%d" % k for k in range(2, T + 1)]


def negative_history(features: Mapping[str, object], T: int, seed: int, n_movies: int = 1001) -> Dict[str, np.ndarray]:
    """The negative samples of the reference's `get_dataset_with_negtive_movie` (DIEN.py:30-47), draw for draw:
    `negtive_userRatedMovie<k>` (int32 [N], k = 2..T) for the feature dict's `userRatedMovie<k>` columns.

    The reference does, on the test file with seed 2021 (:50):
      1. `tmp_df.fillna(0)` - a missing history id becomes 0 (NaN here);
      2. `random.seed(seed)` - the module-level Mersenne Twister, seeded from the int;
      3. `tmp_df.loc[:, 'userRatedMovie2':'userRatedMovie5'].applymap(lambda x: random.sample(
         set(range(0, 1001)) - set([int(x)]), 1)[0])`.
    pandas >= 1.1 runs `applymap` as one `map` per column, columns left to right, rows in order, so the draws
    go column by column.  Python 3.8's `random.sample` turns a set population into `tuple(population)`; a set of
    small ints iterates in ascending order (each int hashes to itself and the table is larger than 1000), so
    that tuple is the sorted list used here (Python 3.11+ rejects a set population).  With n = 999 or 1000
    elements and k = 1, `sample` takes its set-selection branch (n > 21) and returns population[randbelow(n)]
    on both versions: one `_randbelow` per cell, the same words of the generator.  A fresh `random.Random(seed)`
    is the state `random.seed(seed)` gives the module generator.

    Caveat: pandas < 1.1 ran `applymap` through `apply`, which called the function on the first column twice
    (once to infer the result type); under those versions every draw after the first column's is shifted and
    this does not reproduce them."""
    import random
    rng = random.Random(seed)
    pops: Dict[int, list] = {}
    out: Dict[str, np.ndarray] = {}
    for k, key in zip(range(2, T + 1), negative_history_keys(T)):
        col = np.asarray(_as_1d(features, "userRatedMovie%d" % k), np.float64)
        col = np.where(np.isnan(col), 0.0, col)                                  # fillna(0)
        vals = np.empty(col.shape[0], np.int32)
        for i, x in enumerate(col.tolist()):
            x = int(x)
            pop = pops.get(x)
            if pop is None:
                pop = pops[x] = sorted(set(range(0, n_movies)) - {x})
            vals[i] = rng.sample(pop, 1)[0]
        out[key] = vals
    return out


def synthetic_features(spec: ModelSpec, batch: int, seed: int, *, zipf_a: float = 1.05,
                       missing_genre: float = 0.10, uniform_history: bool = False,
                       pad_history: bool = True) -> Dict[str, np.ndarray]:
    """Synthetic MovieLens-shaped feature dict (SURVEY.md section 8d, cfg 2-5).

    Movie ids Zipf(zipf_a) over the vocabulary (or uniform), user ids uniform,
    numerics drawn from the empirical ranges of the bundled data with 2-decimal
    rounding, genres uniform over the 19-word vocabulary with `missing_genre`
    probability of "".  DIN history lengths are uniform in 1..T and the tail is
    0-padded; padding is *included* in the computation, as in the reference
    (SURVEY.md section 8a: `mask_zero=True` has no numerical effect).
    """
    rng = np.random.default_rng(seed)
    B = batch

    # DIN.py:95,125 feeds the movie ids through float32: above 2**24 an id is rounded, and the last few
    # ids of a 10**8 vocabulary round UP to the vocabulary size (out of range in the reference too).
    # Draw only ids whose float32 image is still inside the vocabulary (no change for V <= 2**24).
    top = spec.n_movies
    while int(np.float32(top - 1)) >= spec.n_movies:
        top -= 1

    def movie_ids(n):
        if uniform_history:
            return rng.integers(1, top, size=n, dtype=np.int64)
        # Zipf over ranks 1..V-1 by inverse-CDF on a truncated power law
        u = rng.random(n)
        V = spec.n_movies - 1
        a = zipf_a
        # continuous approximation of truncated zipf: x = ((V^(1-a)-1)u+1)^(1/(1-a))
        x = ((V ** (1.0 - a) - 1.0) * u + 1.0) ** (1.0 / (1.0 - a))
        return np.clip(np.floor(x).astype(np.int64), 1, top - 1)

    f: Dict[str, np.ndarray] = {}
    f["movieId"] = movie_ids(B).astype(np.int32)
    f["userId"] = rng.integers(1, spec.n_users, size=B, dtype=np.int64).astype(np.int32)
    T = spec.hist_len if spec.model in ("din", "dien") else 5
    hist = movie_ids(B * T).reshape(B, T)
    if pad_history:
        lens = rng.integers(1, T + 1, size=B)
        hist[np.arange(T)[None, :] >= lens[:, None]] = 0
    for k in range(T):
        f["userRatedMovie%d" % (k + 1)] = hist[:, k].astype(np.int32)
    r2 = lambda a: np.round(a, 2).astype(np.float32)
    f["releaseYear"] = rng.integers(1926, 1999, size=B).astype(np.int32)
    f["movieRatingCount"] = rng.integers(2, 14617, size=B).astype(np.int32)
    f["movieAvgRating"] = r2(rng.uniform(1.33, 4.45, size=B))
    f["movieRatingStddev"] = r2(rng.uniform(0.49, 1.89, size=B))
    f["userRatingCount"] = rng.integers(2, 101, size=B).astype(np.int32)
    f["userAvgRating"] = r2(rng.uniform(0.5, 5.0, size=B))
    f["userRatingStddev"] = r2(rng.uniform(0.0, 3.18, size=B))
    vocab = np.array(GENRE_VOCAB + ("",), dtype=object)
    for k in (*MOVIE_GENRE_KEYS, *USER_GENRE_KEYS):
        g = rng.integers(0, len(GENRE_VOCAB), size=B)
        g[rng.random(B) < missing_genre] = len(GENRE_VOCAB)
        f[k] = vocab[g]
    return f
