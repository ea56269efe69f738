"""CPU oracle of the reference's sample builder, `FeatureEngForRecModel.scala:21-130` (ratings.csv + movies.csv ->
the 27-column sample rows every model here reads).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

Each step restates one statement of the Scala (line numbers in the comments); DESIGN.md section 4.11 gives the
semantics and the two rules Spark leaves open, which the device path shares:

* rows of one user with equal timestamps keep ratings.csv file order;
* genres of equal count keep the iteration order of the Scala 2.11 `mutable.HashMap` the UDF counts them in
  (`scala_hashmap_keys` is that table, entry by entry; `_genre_order_keys` is its closed form, which the window
  code and the device use).

Averages come from exact integer sums (ratings are half-stars, years are integers), so they do not depend on the
order of the rows.  A user window's standard deviations follow Spark's own update (`_welford_stddev`) in window
order: the window's order is defined, and the rounding of that update decides some HALF_EVEN ties (a variance of
exactly 49/64 prints as 0.87, not 0.88).  A movie's rows are aggregated in an order Spark does not define, so its
standard deviation is the exact sqrt(Q / (4 n (n - 1))) with Q = n S2 - S1^2 in half-stars: one correctly rounded
division of two integers below 2^53.

The window code runs on user-aligned chunks of the sorted rows, so memory stays bounded at ML-20M sizes.
"""
from __future__ import annotations

import re
from decimal import ROUND_HALF_EVEN, Decimal
from typing import Dict, List, Sequence

import numpy as np

WINDOW = 100                 # rowsBetween(-100, -1)
MAX_GENRE_WORDS = 24         # one HashMap resize (16 -> 32 buckets at the 13th key); a second would come at the 25th
DEFAULT_YEAR = 1990          # extractReleaseYearUdf's default
CHUNK_ROWS = 1 << 20

COLUMNS = ("movieId", "userId", "rating", "timestamp", "label", "releaseYear", "movieGenre1", "movieGenre2",
           "movieGenre3", "movieRatingCount", "movieAvgRating", "movieRatingStddev", "userRatedMovie1",
           "userRatedMovie2", "userRatedMovie3", "userRatedMovie4", "userRatedMovie5", "userRatingCount",
           "userAvgReleaseYear", "userReleaseYearStddev", "userAvgRating", "userRatingStddev", "userGenre1",
           "userGenre2", "userGenre3", "userGenre4", "userGenre5")

_JAVA_WS = "".join(chr(c) for c in range(33))      # String.trim strips every char <= ' '
_JAVA_INT = re.compile(r"[+-]?[0-9]+\Z")


# ----------------------------------------------------------------------------------------------- the title UDF
def release_year(title) -> int:
    """extractReleaseYearUdf (:36-44): `title.trim.substring(title.length - 5, title.length - 1).toInt`, 1990 for a
    null title or a trimmed title shorter than 6.  The substring takes the *untrimmed* length; where Java would
    throw (index past the trimmed string, or not an integer) this raises ValueError, as the Spark job would fail."""
    if title is None:
        return DEFAULT_YEAR
    t = title.strip(_JAVA_WS)
    if len(t) < 6:
        return DEFAULT_YEAR
    b, e = len(title) - 5, len(title) - 1
    if e > len(t):
        raise ValueError("title %r: substring(%d, %d) past the trimmed length %d" % (title, b, e, len(t)))
    s = t[b:e]
    if not _JAVA_INT.match(s):
        raise ValueError("title %r: %r is not an integer" % (title, s))
    return int(s)


# ------------------------------------------------------------------------------------------- format_number(x, 2)
def format2_hundredths(x: np.ndarray) -> np.ndarray:
    """`format_number(x, 2)`: java.text.DecimalFormat, HALF_EVEN on the double's exact binary value -> the integer
    k of hundredths it prints (int64).  x must be finite and >= 0."""
    x = np.asarray(x, np.float64)
    u, inv = np.unique(x, return_inverse=True)
    q = Decimal("0.01")
    k = np.array([int(Decimal(float(v)).quantize(q, rounding=ROUND_HALF_EVEN) * 100) for v in u], np.int64)
    return k[inv].reshape(x.shape)


def hundredths_to_f32(k: np.ndarray) -> np.ndarray:
    """The float32 nearest k/100: what float32(float("<k/100 as text>")) gives for every k < 10^5."""
    return np.asarray(k, np.int64).astype(np.float32) / np.float32(100)


def format2_text(v: float) -> str:
    """DecimalFormat "#,###,##0.00" of a two-decimal value (the grouping comma included)."""
    return "{:,.2f}".format(float(v))


# ----------------------------------------------------------------------------- the UDF's Scala 2.11 HashMap order
def java_string_hash(s: str) -> int:
    """java.lang.String.hashCode over UTF-16 code units, as a signed 32-bit int."""
    b = s.encode("utf-16-le")
    h = 0
    for i in range(0, len(b), 2):
        h = (31 * h + (b[i] | (b[i + 1] << 8))) & 0xFFFFFFFF
    return h - (1 << 32) if h >= 1 << 31 else h


def _hash_bucket(h: int, table_len: int) -> int:
    """scala.collection.mutable.HashTable.index: byteswap32, rotate right by the seed (bitCount(15) = 4, fixed at
    construction), then the top log2(table_len) bits."""
    m = 0xFFFFFFFF
    hc = (h * 0x9E3775CD) & m
    hc = int.from_bytes(hc.to_bytes(4, "little"), "big")          # Integer.reverseBytes
    hc = (hc * 0x9E3775CD) & m
    rot = ((hc >> 4) | (hc << 28)) & m
    bits = table_len.bit_length() - 1
    return rot >> (32 - bits)


def genre_buckets(hashes: Sequence[int]):
    """(bucket in the 16-slot table, bucket in the 32-slot table) of each genre word's String.hashCode."""
    b16 = np.array([_hash_bucket(int(h), 16) for h in hashes], np.int64)
    b32 = np.array([_hash_bucket(int(h), 32) for h in hashes], np.int64)
    return b16, b32


def scala_hashmap_keys(words: Sequence[str]) -> List[str]:
    """Keys of a Scala 2.11 `mutable.HashMap[String, Int]` after inserting `words` (first occurrences matter), in its
    iteration order: entries go to the head of their bucket; above 12 entries the 16-slot table is rehashed into
    32 slots, old buckets high to low, each bucket head first; iteration runs buckets high to low, head first."""
    table: List[list] = [[] for _ in range(16)]
    size = 0
    seen = set()
    for w in words:
        if w in seen:
            continue
        seen.add(w)
        table[_hash_bucket(java_string_hash(w), len(table))].insert(0, w)
        size += 1
        if size > len(table) * 3 // 4:
            old, table = table, [[] for _ in range(2 * len(table))]
            for i in range(len(old) - 1, -1, -1):
                for e in old[i]:
                    table[_hash_bucket(java_string_hash(e), len(table))].insert(0, e)
    return [w for b in reversed(table) for w in b]


def _genre_order_keys(ins, n_distinct, b16, b32):
    """Closed form of scala_hashmap_keys: a key per present genre, ascending in iteration order.  `ins` is the
    genre's insertion rank (0 = first inserted), `n_distinct` the number of keys, b16 / b32 its buckets."""
    small = ((15 - b16) << 8) | (255 - ins)
    post = ins >= 13                                                     # inserted after the resize
    big = ((31 - b32) << 16) | np.where(post, 255 - ins, (1 << 15) | (b16 << 8) | ins)
    return np.where(n_distinct <= 12, small, big)


# ------------------------------------------------------------------------------------------------ the job itself
def movie_table(movies: Dict[str, Sequence], n_slots: int):
    """movies.csv -> per movie id: release year, genre word indices in string order (-1 padded), and the genre
    words (distinct words of the genres column in first-appearance order).  A movie absent from movies.csv gets
    1990 and no genres (the left join leaves title and genres null)."""
    words: Dict[str, int] = {}
    lists = []
    for g in movies["genres"]:
        lists.append([words.setdefault(w, len(words)) for w in g.split("|")] if g is not None else [])
    if len(words) > MAX_GENRE_WORDS:
        raise ValueError("%d distinct genre words; at most %d are supported" % (len(words), MAX_GENRE_WORDS))
    L = max([len(x) for x in lists] + [1])
    year = np.full(n_slots, DEFAULT_YEAR, np.int64)
    genres = np.full((n_slots, L), -1, np.int64)
    for mid, title, gl in zip(np.asarray(movies["movieId"]).tolist(), movies["title"], lists):
        year[mid] = release_year(title)
        genres[mid, :len(gl)] = gl
    return year, genres, list(words)


def _stddev(n, s1, s2, scale):
    """stddev_samp from exact integer moments; n < 2 gives 0 (NaN / null, then na.fill(0))."""
    nn = np.maximum(n, 2).astype(np.int64)
    q = (n.astype(np.int64) * s2 - s1 * s1).astype(np.float64)
    var = q / (scale * nn * (nn - 1)).astype(np.float64)
    return np.where(n >= 2, np.sqrt(var), 0.0)


def movie_features(count, sum_half, sum_half2):
    """addMovieFeatures (:59-63) from a movie's rating moments in half-stars: the hundredths format_number prints
    for avg(rating) and for stddev(rating) (na.fill(0) for a single rating)."""
    count, sum_half, sum_half2 = (np.asarray(a, np.int64) for a in (count, sum_half, sum_half2))
    avg = np.where(count > 0, (sum_half / 2.0) / np.maximum(count, 1), 0.0)
    return format2_hundredths(avg), format2_hundredths(_stddev(count, sum_half, sum_half2, 4))


def _welford_stddev(x, lo, i):
    """stddev_samp over the window rows lo .. i - 1 in window order, as Spark's CentralMomentAgg updates it (one
    double rounding per operation, no fused multiply-add); the frame is re-aggregated for every row."""
    n = np.zeros(len(i))
    avg = np.zeros(len(i))
    m2 = np.zeros(len(i))
    for t in range(WINDOW):
        idx = lo + t
        act = idx < i
        v = x[np.minimum(idx, len(x) - 1)]
        new_n = n + 1.0
        delta = v - avg
        delta_n = delta / new_n
        avg = np.where(act, avg + delta_n, avg)
        m2 = np.where(act, m2 + delta * (delta - delta_n), m2)
        n = np.where(act, new_n, n)
    return np.where(n >= 2, np.sqrt(m2 / np.maximum(n - 1.0, 1.0)), 0.0)


def _windows(S, lo_all, a, b, year_of, genres_of, G, b16, b32, out):
    """User windows of sorted rows [a, b) (a and b are user starts)."""
    M = b - a
    lo = lo_all[a:b] - a
    i = np.arange(M)
    n = i - lo
    h, mv = S["half"][a:b], S["movie"][a:b]
    y = year_of[mv]
    pos = h >= 7                                                          # label: rating >= 3.5
    pre = lambda v: np.concatenate([[0], np.cumsum(v, dtype=np.int64)])
    win = lambda v: (lambda p: p[i] - p[lo])(pre(v))
    s1, y1 = win(h), win(y)
    nz = np.maximum(n, 1)
    out["userRatingCount"][a:b] = n
    out["userAvgRating_k"][a:b] = format2_hundredths(np.where(n > 0, (s1 / 2.0) / nz, 0.0))
    out["userRatingStddev_k"][a:b] = format2_hundredths(_welford_stddev(h / 2.0, lo, i))
    out["userAvgReleaseYear"][a:b] = np.where(n > 0, np.trunc(y1 / nz), 0.0)      # avg(...).cast(IntegerType)
    out["userReleaseYearStddev_k"][a:b] = format2_hundredths(_welford_stddev(y.astype(np.float64), lo, i))
    # collect_list(positive movieId) over the window, reversed, getItem(0..4)
    cp = pre(pos)
    plist = np.flatnonzero(pos)
    for k in range(5):
        j = cp[i] - 1 - k
        ok = j >= 0
        src = plist[np.where(ok, j, 0)] if plist.size else np.zeros(M, np.int64)
        ok &= src >= lo
        out["userRatedMovie%d" % (k + 1)][a:b] = np.where(ok, mv[src] if plist.size else 0, 0)
    # extractGenres over collect_list(positive genres): counts, then the HashMap's order, stable by count desc
    gl = genres_of[mv]                                                     # [M, L]
    L = gl.shape[1]
    has = np.zeros((M, G), np.int64)
    gpos = np.full((M, G), L, np.int64)                                   # first position of g in the row's list
    for p in range(L - 1, -1, -1):
        g = gl[:, p]
        r = np.flatnonzero(pos & (g >= 0))
        np.add.at(has, (r, g[r]), 1)
        gpos[r, g[r]] = p
    cnt_pre = np.concatenate([np.zeros((1, G), np.int64), np.cumsum(has, axis=0)])
    first = np.where(has > 0, i[:, None], M)
    nxt = np.concatenate([np.minimum.accumulate(first[::-1], axis=0)[::-1], np.full((1, G), M)])
    cnt = cnt_pre[i] - cnt_pre[lo]                                        # [M, G]
    frow = nxt[lo]                                                        # first window row holding g
    present = cnt > 0
    fkey = np.where(present, frow * (L + 1) + gpos[np.minimum(frow, M - 1), np.arange(G)[None, :]], 1 << 40)
    ins = np.argsort(np.argsort(fkey, axis=1, kind="stable"), axis=1, kind="stable")
    nd = present.sum(axis=1, keepdims=True)
    ok = _genre_order_keys(ins, nd, b16[None, :], b32[None, :])
    key = np.where(present, ((1000 - cnt) << 24) | ok, 1 << 50)
    order = np.argsort(key, axis=1, kind="stable")[:, :5]                 # fewer than 5 columns if G < 5
    got = np.take_along_axis(present, order, axis=1)
    for k in range(5):
        out["userGenre%d_i" % (k + 1)][a:b] = np.where(got[:, k], order[:, k], -1) if k < G else -1


def build_samples(ratings: Dict[str, np.ndarray], movies: Dict[str, Sequence]) -> Dict[str, np.ndarray]:
    """ratings: userId, movieId, rating (float, as read), timestamp (int > 0); movies: movieId, title, genres.
    Returns the kept rows in ratings.csv order, keyed and typed as `features.load_samples_csv` returns them."""
    user = np.asarray(ratings["userId"], np.int64)
    movie = np.asarray(ratings["movieId"], np.int64)
    rating = np.asarray(ratings["rating"], np.float64)
    ts = np.asarray(ratings["timestamp"], np.int64)
    N = user.shape[0]
    half = np.rint(rating * 2).astype(np.int64)
    n_slots = int(max(movie.max(initial=0), np.asarray(movies["movieId"]).max(initial=0))) + 1
    year_of, genres_of, words = movie_table(movies, n_slots)
    G = max(len(words), 1)
    hashes = [java_string_hash(w) for w in words] or [0]
    b16, b32 = genre_buckets(hashes)

    # addMovieFeatures (:59-63): count, format_number(avg), format_number(stddev, na.fill(0)) over all ratings
    mc = np.bincount(movie, minlength=n_slots)
    m1 = np.bincount(movie, weights=half, minlength=n_slots).astype(np.int64)
    m2 = np.bincount(movie, weights=half * half, minlength=n_slots).astype(np.int64)
    m_avg_k, m_std_k = movie_features(mc, m1, m2)

    # Window.partitionBy("userId").orderBy(col("timestamp")): timestamp is a string, ties in file order
    digits = np.floor(np.log10(ts.astype(np.float64))).astype(np.int64) + 1
    digits += (ts >= 10 ** digits).astype(np.int64) - (ts < 10 ** (digits - 1)).astype(np.int64)
    aligned = ts * 10 ** (10 - digits)
    order = np.lexsort((np.arange(N), digits, aligned, user))
    S = {"half": half[order], "movie": movie[order]}
    su = user[order]
    start = np.flatnonzero(np.r_[True, su[1:] != su[:-1]])
    seg = np.repeat(start, np.diff(np.r_[start, N]))
    lo_all = np.maximum(seg, np.arange(N) - WINDOW)

    w = {k: np.zeros(N, np.int64) for k in ("userRatingCount", "userAvgRating_k", "userRatingStddev_k",
                                              "userReleaseYearStddev_k", "userRatedMovie1", "userRatedMovie2",
                                              "userRatedMovie3", "userRatedMovie4", "userRatedMovie5",
                                              "userGenre1_i", "userGenre2_i", "userGenre3_i", "userGenre4_i",
                                              "userGenre5_i")}
    w["userAvgReleaseYear"] = np.zeros(N, np.float64)
    bounds = sorted(set(int(seg[c]) for c in range(0, N, CHUNK_ROWS)) | {N})     # chunk edges on user starts
    for a, b in zip(bounds[:-1], bounds[1:]):
        _windows(S, lo_all, a, b, year_of, genres_of, G, b16, b32, w)

    back = np.empty(N, np.int64)
    back[order] = np.arange(N)
    keep = w["userRatingCount"][back] > 1                                 # .filter(userRatingCount > 1)
    rows = back[keep]
    fi = np.flatnonzero(keep)
    mv = movie[fi]
    word = np.array(words + [""], dtype=object)
    gname = lambda idx: word[np.where(idx >= 0, idx, len(words))]
    out: Dict[str, np.ndarray] = {
        "movieId": mv.astype(np.int32), "userId": user[fi].astype(np.int32),
        "rating": (half[fi] / 2.0).astype(np.float32), "timestamp": ts[fi].astype(np.int32),
        "label": (half[fi] >= 7).astype(np.int32), "releaseYear": year_of[mv].astype(np.int32)}
    for k in range(3):
        out["movieGenre%d" % (k + 1)] = gname(genres_of[mv, k] if genres_of.shape[1] > k else np.full(len(mv), -1))
    out["movieRatingCount"] = mc[mv].astype(np.int32)
    out["movieAvgRating"] = hundredths_to_f32(m_avg_k[mv])
    out["movieRatingStddev"] = hundredths_to_f32(m_std_k[mv])
    for k in range(1, 6):
        out["userRatedMovie%d" % k] = w["userRatedMovie%d" % k][rows].astype(np.int32)
    out["userRatingCount"] = w["userRatingCount"][rows].astype(np.int32)
    out["userAvgReleaseYear"] = w["userAvgReleaseYear"][rows].astype(np.float32)
    out["userReleaseYearStddev"] = hundredths_to_f32(w["userReleaseYearStddev_k"][rows])
    out["userAvgRating"] = hundredths_to_f32(w["userAvgRating_k"][rows])
    out["userRatingStddev"] = hundredths_to_f32(w["userRatingStddev_k"][rows])
    for k in range(1, 6):
        out["userGenre%d" % k] = gname(w["userGenre%d_i" % k][rows])
    return {c: out[c] for c in COLUMNS}
