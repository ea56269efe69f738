"""CPU oracle of the reference's FeatureEngineering job (`OFF/featureeng/FeatureEngineering.scala`) and of the
tail of FeatureEngForRecModel (`splitAndSaveTrainingTestSamples`, `:176-188`, and its timestamp twin, `:190-205`).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

DESIGN.md section 4.16 gives the semantics.  Spark 2.4.3 / Scala 2.11 internals are restated from memory, class by
class; the reference ships no output of this job, so the hand-worked known answers in the tests are what hold them:

* `QuantileSummaries` is Spark's class literally (head buffer, `withHeadBufferInserted`, `compress`, `merge`,
  `query`), and `spark_approx_quantile` runs it over partitions as `StatFunctions.multipleApproxQuantiles` does
  (fold each partition, then `s1.compress().merge(s2.compress())`).
* `one_summary_quantiles` is the answer when every value goes through one summary with one head buffer: what the
  device computes.  `one_summary_closed_form` is the device's jump-ahead form of the same compress walk.
* `hash_trie_keys` is a Scala 2.11 `immutable.HashMap` (a hash trie over `improve(hashCode)`, 5 bits a level from
  the low bits) built entry by entry; `trie_order_key` is its closed form, which the device sorts by.
* `split_samples` / `split_samples_by_timestamp` draw from counter-based splitmix streams (collab.random_split's
  uniforms, one derived stream for the sample and one for the split).
"""
from __future__ import annotations

import math
from decimal import Decimal
from fractions import Fraction
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .feature_eng import java_string_hash

DEFAULT_HEAD_SIZE = 50000           # QuantileSummaries.defaultHeadSize
DEFAULT_COMPRESS_THRESHOLD = 10000  # QuantileSummaries.defaultCompressThreshold
_M32 = 0xFFFFFFFF
_M64 = (1 << 64) - 1


# ------------------------------------------------------------------------------------ Spark's QuantileSummaries
class QuantileSummaries:
    """org.apache.spark.sql.catalyst.util.QuantileSummaries (2.4.3).  `sampled` is a list of [value, g, delta].
    `target_error_ceil` picks the query's rule: `math.ceil(relativeError * count)` (the rule implemented here) or
    the unrounded `relativeError * count`."""

    def __init__(self, relative_error: float, compress_threshold: int = DEFAULT_COMPRESS_THRESHOLD,
                 sampled=None, count: int = 0, head_size: int = DEFAULT_HEAD_SIZE, target_error_ceil: bool = True):
        self.relative_error = float(relative_error)
        self.compress_threshold = compress_threshold
        self.sampled: List[list] = list(sampled or [])
        self.count = count
        self.head: List[float] = []
        self.head_size = head_size
        self.target_error_ceil = target_error_ceil

    def _new(self, sampled, count):
        return QuantileSummaries(self.relative_error, self.compress_threshold, sampled, count, self.head_size,
                                 self.target_error_ceil)

    def insert(self, x: float) -> "QuantileSummaries":
        self.head.append(float(x))
        if len(self.head) >= self.head_size:
            result = self._with_head_buffer_inserted()
            return result.compress() if len(result.sampled) >= self.compress_threshold else result
        return self

    def _with_head_buffer_inserted(self) -> "QuantileSummaries":
        if not self.head:
            return self
        current = self.count
        srt = sorted(self.head)
        new: List[list] = []
        si = 0
        for oi, x in enumerate(srt):
            while si < len(self.sampled) and self.sampled[si][0] <= x:
                new.append(self.sampled[si])
                si += 1
            current += 1
            if not new or (si == len(self.sampled) and oi == len(srt) - 1):
                delta = 0
            else:
                delta = int(math.floor(2 * self.relative_error * current))
            new.append([x, 1, delta])
        new.extend(self.sampled[si:])
        return self._new(new, current)

    def compress(self) -> "QuantileSummaries":
        ins = self._with_head_buffer_inserted()
        return self._new(compress_immut(ins.sampled, 2 * self.relative_error * ins.count), ins.count)

    def merge(self, other: "QuantileSummaries") -> "QuantileSummaries":
        assert not self.head and not other.head, "compress before merge"
        if other.count == 0:
            return self._new(self.sampled, self.count)
        if self.count == 0:
            return other._new(other.sampled, other.count)
        res = sorted(self.sampled + other.sampled, key=lambda s: s[0])          # sortBy: stable
        comp = compress_immut(res, 2 * self.relative_error * self.count)      # this.count, as 2.4.3 has it
        return other._new(comp, other.count + self.count)

    def query(self, quantile: float) -> Optional[float]:
        assert 0.0 <= quantile <= 1.0
        assert not self.head, "query an uncompressed summary"
        return query_sampled(self.sampled, self.count, quantile, self.relative_error, self.target_error_ceil)


def compress_immut(samples: Sequence[list], merge_threshold: float) -> List[list]:
    """QuantileSummaries.compressImmut: from the last sample down to the second, merge a sample into the current
    head while sample.g + head.g + head.delta < mergeThreshold; the minimum is kept apart."""
    if not samples:
        return []
    res: List[list] = []
    head = list(samples[-1])
    i = len(samples) - 2
    while i >= 1:
        s = samples[i]
        if s[1] + head[1] + head[2] < merge_threshold:
            head[1] += s[1]
        else:
            res.append(head)
            head = list(s)
        i -= 1
    res.append(head)
    if samples[0][0] <= head[0] and len(samples) > 1:
        res.append(list(samples[0]))
    res.reverse()
    return res


def query_sampled(sampled, count, quantile, eps, target_error_ceil=True):
    """QuantileSummaries.query over compressed samples."""
    if not sampled:
        return None
    if quantile <= eps:
        return sampled[0][0]
    if quantile >= 1 - eps:
        return sampled[-1][0]
    rank = int(math.ceil(quantile * count))
    target = float(math.ceil(eps * count)) if target_error_ceil else eps * count
    min_rank = 0
    for v, g, d in sampled[:-1]:
        min_rank += g
        max_rank = min_rank + d
        if max_rank - target <= rank and rank <= min_rank + target:
            return v
    return sampled[-1][0]


def spark_approx_quantile(partitions: Sequence[Sequence[float]], probabilities: Sequence[float],
                          relative_error: float, target_error_ceil: bool = True,
                          head_size: int = DEFAULT_HEAD_SIZE) -> List[float]:
    """Dataset.stat.approxQuantile over `partitions`: each partition folds its values into a fresh summary
    (`insert`), then the partitions merge left to right as `s1.compress().merge(s2.compress())` (Spark's merge order
    is its tasks' completion order; the result may depend on it).  A lone partition is compressed before the query.
    NaN values are rejected."""
    summaries = []
    for part in partitions:
        s = QuantileSummaries(relative_error, head_size=head_size, target_error_ceil=target_error_ceil)
        for x in part:
            if math.isnan(x):
                raise ValueError("NaN value")
            s = s.insert(x)
        summaries.append(s)
    acc = summaries[0]
    for s in summaries[1:]:
        acc = acc.compress().merge(s.compress())
    acc = acc.compress()
    return [acc.query(p) for p in probabilities]


# ------------------------------------------------------------------------------- the one-summary answer (device)
def one_summary_samples(values: np.ndarray, relative_error: float) -> Tuple[np.ndarray, list, int]:
    """Every value through one summary with one head buffer: sort (Double total order), `withHeadBufferInserted`
    (delta = floor(2 eps (i + 1)) except at both ends), then `compressImmut` with mergeThreshold 2 eps n.
    Returns (sorted values, compressed samples, n)."""
    v = np.asarray(values, np.float64)
    if np.isnan(v).any():
        raise ValueError("NaN value")
    srt = v[np.argsort(_total_order_keys(v), kind="stable")]
    n = len(srt)
    eps = float(relative_error)
    samples = [[float(x), 1, 0 if i == 0 or i == n - 1 else int(math.floor(2 * eps * (i + 1)))]
               for i, x in enumerate(srt.tolist())]
    return srt, compress_immut(samples, 2 * eps * n), n


def one_summary_quantiles(values, probabilities, relative_error, target_error_ceil=True) -> np.ndarray:
    """approxQuantile as one summary gives it (`one_summary_samples`, then `query`)."""
    _, sampled, n = one_summary_samples(values, relative_error)
    if n == 0:
        raise ValueError("no values")
    return np.array([query_sampled(sampled, n, float(p), float(relative_error), target_error_ceil)
                     for p in probabilities], np.float64)


def one_summary_closed_form(n: int, relative_error: float) -> List[Tuple[int, int, int]]:
    """The compress walk of `one_summary_samples` in the device's jump-ahead form, as (sorted index, g, delta),
    ascending.  Every sample starts with g = 1, so a head at sorted index j with delta d absorbs
    m = max(0, ceil(T - 2 - d)) samples below it (at most j - 1), T = 2 eps n."""
    eps = float(relative_error)
    T = 2 * eps * n

    def delta(j):
        return 0 if j == 0 or j == n - 1 else int(math.floor(2 * eps * (j + 1)))

    out = []
    j = n - 1
    while True:
        d = delta(j)
        x = T - float(d + 2)
        m = min(int(math.ceil(x)) if x > 0 else 0, max(j - 1, 0))
        out.append((j, 1 + m, d))
        j = j - m - 1
        if j < 1:
            break
    if n > 1:
        out.append((0, 1, 0))
    out.reverse()
    return out


def one_summary_segments(n: int, relative_error: float) -> List[Tuple[int, int, int]]:
    """The device's form of the same walk (fj_compress_kernel): delta, hence the take t = ceil(T - 2 - d), is
    constant over runs of sorted indices, so the heads of a run are an arithmetic progression of stride t + 1 and
    the walk takes one step per run (or per head, near the ends).  Returns (sorted index, g, delta), ascending."""
    e2 = 2.0 * float(relative_error)
    T = e2 * n

    def delta(j):
        return 0 if j == 0 or j == n - 1 else int(math.floor(e2 * float(j + 1)))

    heads = []
    j = n - 1
    while True:
        d = delta(j)
        x = T - float(d + 2)
        t = int(math.ceil(x)) if x > 0 else 0
        if 1 <= j <= n - 2 and t <= j - 1:
            a, b = 1, j
            while a < b:
                mid = (a + b) // 2
                if delta(mid) >= d:
                    b = mid
                else:
                    a = mid + 1
            lo = max(a, t + 1)
            count = (j - lo) // (t + 1) + 1
            heads.extend((j - (t + 1) * k, 1 + t, d) for k in range(count))
            j -= count * (t + 1)
        else:
            take = min(t, max(j - 1, 0))
            heads.append((j, 1 + take, d))
            j -= take + 1
        if j < 1:
            break
    if n > 1:
        heads.append((0, 1, 0))
    return heads[::-1]


def _total_order_keys(v: np.ndarray) -> np.ndarray:
    """java.lang.Double.compare's order (-0.0 < 0.0) as uint64 keys."""
    b = np.ascontiguousarray(v, np.float64).view(np.uint64)
    neg = (b >> np.uint64(63)) == 1
    return np.where(neg, ~b, b | np.uint64(1 << 63))


# ------------------------------------------------------------------------------- QuantileDiscretizer, Bucketizer
def discretizer_probabilities(num_buckets: int) -> List[float]:
    """`(0.0 to 1.0 by 1.0 / numBuckets).toArray`, a Scala 2.11 NumericRange[Double]: length
    (BigDecimal(1.0) quot BigDecimal(step)) + 1, where BigDecimal(step) is the decimal Double.toString prints (the
    shortest one that reads back, as repr gives it), and element k = 0.0 + step * k.  When that decimal exceeds
    1 / numBuckets the range ends one step short of 1.0 (numBuckets 11 gives 11 elements, the last 10 / 11)."""
    step = 1.0 / num_buckets
    count = int(Fraction(1) // Fraction(Decimal(repr(step)))) + 1
    return [0.0 + step * float(k) for k in range(count)]


def discretizer_splits(values, num_buckets: int, relative_error: float = 0.001,
                       target_error_ceil: bool = True) -> np.ndarray:
    """QuantileDiscretizer.fit: approxQuantile at `discretizer_probabilities`, the ends replaced by -inf and +inf,
    then `distinct` (Double.equals: bit equality), keeping order; the Bucketizer requires >= 3 strictly increasing
    splits."""
    if num_buckets < 2:
        raise ValueError("numBuckets must be >= 2")
    probs = discretizer_probabilities(num_buckets)
    q = one_summary_quantiles(values, probs, relative_error, target_error_ceil)
    q[0], q[-1] = -np.inf, np.inf
    seen, out = set(), []
    for x in q.tolist():
        key = np.float64(x).view(np.uint64).item()
        if key not in seen:
            seen.add(key)
            out.append(x)
    s = np.array(out, np.float64)
    if len(s) < 3 or not np.all(s[:-1] < s[1:]):
        raise ValueError("splits %r are not >= 3 strictly increasing values" % (s,))
    return s


def bucketize(splits, values) -> np.ndarray:
    """Bucketizer.binarySearchForBuckets with handleInvalid "error": a value equal to the last split goes to the
    last bucket; otherwise java.util.Arrays.binarySearch (Double total order): a value on a split goes to the bucket
    above it.  NaN or a value outside [splits[0], splits[-1]] raises ValueError."""
    s = np.asarray(splits, np.float64)
    v = np.asarray(values, np.float64)
    if np.isnan(v).any():
        raise ValueError("NaN value")
    sk, vk = _total_order_keys(s), _total_order_keys(v)
    last = v == s[-1]
    if (~last & ((vk < sk[0]) | (vk > sk[-1]))).any():
        raise ValueError("value outside the splits")
    idx = np.searchsorted(sk, vk, side="right") - 1
    return np.where(last, len(s) - 2, idx).astype(np.float64)


def min_max_scale(values, fit_min=None, fit_max=None):
    """MinMaxScaler (min 0, max 1): (x - Emin) / (Emax - Emin), 0.5 when the range is 0; E from the data unless
    given.  Returns (scaled, Emin, Emax).  NaN raises ValueError."""
    v = np.asarray(values, np.float64)
    if np.isnan(v).any():
        raise ValueError("NaN value")
    if fit_min is None:
        k = _total_order_keys(v)
        fit_min, fit_max = float(v[np.argmin(k)]), float(v[np.argmax(k)])
    rng = fit_max - fit_min
    out = (v - fit_min) / rng if rng != 0 else np.full(v.shape, 0.5)
    return out, fit_min, fit_max


# --------------------------------------------------------------------------------------- StringIndexer, 2.11 trie
def improve(h: int) -> int:
    """scala.collection.immutable.HashMap.improve (2.11), on a 32-bit int; returned unsigned."""
    h &= _M32
    h = (h + (~(h << 9) & _M32)) & _M32
    h ^= h >> 14
    h = (h + (h << 4)) & _M32
    return h ^ (h >> 10)


def trie_order_key(hash_code: int) -> int:
    """Closed form of the trie's iteration order: improve(hashCode) read as 5-bit digits from the low bits, the
    lowest digit most significant (35 bits)."""
    h = improve(hash_code)
    k = 0
    for level in range(7):
        k = (k << 5) | ((h >> (5 * level)) & 31)
    return k


def hash_trie_keys(words: Sequence[str]) -> List[str]:
    """Keys of a Scala 2.11 `immutable.HashMap[String, _]` built by adding `words` one by one, in iteration order.
    A HashTrieMap node holds its children in ascending 5-bit index, (improve(hash) >>> level) & 31; two keys that
    share the index at a level go one level down.  Full-hash collisions (a HashMapCollision1) raise."""
    root: dict = {}

    def add(node, h, w, level):
        i = (h >> level) & 31
        cur = node.get(i)
        if cur is None:
            node[i] = (h, w)
        elif isinstance(cur, dict):
            add(cur, h, w, level + 5)
        elif cur[1] == w:
            return
        elif cur[0] == h:
            raise ValueError("hash collision between %r and %r" % (cur[1], w))
        else:
            sub: dict = {}
            add(sub, cur[0], cur[1], level + 5)
            add(sub, h, w, level + 5)
            node[i] = sub

    for w in words:
        add(root, improve(java_string_hash(w)), w, 0)

    out: List[str] = []

    def walk(node):
        for i in sorted(node):
            c = node[i]
            walk(c) if isinstance(c, dict) else out.append(c[1])

    walk(root)
    return out


def string_indexer_labels(tokens: Sequence[str]) -> Tuple[List[str], List[int]]:
    """StringIndexer.fit (frequencyDesc): countByValue's map in iteration order, then a stable sort by descending
    count.  Returns (labels, counts)."""
    counts: Dict[str, int] = {}
    for t in tokens:
        counts[t] = counts.get(t, 0) + 1
    order = hash_trie_keys(list(counts))
    labels = sorted(order, key=lambda w: -counts[w])
    return labels, [counts[w] for w in labels]


# ---------------------------------------------------------------------------------------------- the job's parts
def one_hot(movie_ids) -> Tuple[np.ndarray, int]:
    """OneHotEncoderEstimator(dropLast = false) on movieId cast to int: (index per row, category count max + 1)."""
    ids = np.asarray(movie_ids, np.int64)
    return ids.astype(np.int32), int(ids.max()) + 1


def multi_hot(movie_ids, genres: Sequence[str]):
    """multiHotEncoderExample: StringIndexer over the `|`-split genre words, then per movie (ascending id) the
    sorted label indices of its words.  Returns (labels, counts, movie ids, CSR offsets, indices)."""
    lists = [g.split("|") for g in genres]
    for mid, gl in zip(np.asarray(movie_ids).tolist(), lists):
        if len(set(gl)) != len(gl):
            raise ValueError("movie %d lists a genre twice" % mid)
    labels, counts = string_indexer_labels([w for gl in lists for w in gl])
    index = {w: k for k, w in enumerate(labels)}
    ids = np.asarray(movie_ids, np.int64)
    order = np.argsort(ids, kind="stable")
    offsets, indices = [0], []
    for r in order.tolist():
        indices.extend(sorted(index[w] for w in lists[r]))
        offsets.append(len(indices))
    return labels, counts, ids[order].astype(np.int32), np.array(offsets, np.int64), np.array(indices, np.int32)


def rating_features_from_moments(count, sum_half, sum_half2):
    """ratingFeatures' groupBy from each movie's exact half-star moments: rows of movies with a rating, ascending
    id: (movie ids, count int64, avg float64, var_samp float64 - NaN for null at one rating).  avg = S1 / (2n) and
    var = Q / (4 n (n - 1)), Q = n S2 - S1^2, each one correctly rounded division of exact integers."""
    c, s1, s2 = (np.asarray(a, np.int64) for a in (count, sum_half, sum_half2))
    ids = np.flatnonzero(c > 0)
    n, a, b = c[ids], s1[ids], s2[ids]
    avg = (a.astype(np.float64) * 0.5) / n.astype(np.float64)
    q = (n * b - a * a).astype(np.float64)
    den = (4 * n * np.maximum(n - 1, 1)).astype(np.float64)
    var = np.where(n >= 2, q / den, np.nan)
    return ids.astype(np.int32), n, avg, var


def rating_features(movie_id, half):
    """rating_features_from_moments over ratings (movie id, rating in half-stars)."""
    m = np.asarray(movie_id, np.int64)
    h = np.asarray(half, np.int64)
    slots = int(m.max()) + 1
    return rating_features_from_moments(np.bincount(m, minlength=slots), np.bincount(m, h, slots).astype(np.int64),
                                        np.bincount(m, h * h, slots).astype(np.int64))


def feature_engineering(movie_id_ratings, half, num_buckets: int = 100, relative_error: float = 0.001):
    """The ratingFeatures pipeline: the groupBy, then QuantileDiscretizer on ratingCount and MinMaxScaler on
    avgRating.  Returns (ids, count, avg, var, bucket, scaled avg, splits)."""
    ids, n, avg, var = rating_features(movie_id_ratings, half)
    splits = discretizer_splits(n.astype(np.float64), num_buckets, relative_error)
    return ids, n, avg, var, bucketize(splits, n.astype(np.float64)), min_max_scale(avg)[0], splits


# ------------------------------------------------------------------------------------------------ sample, split
def splitmix(x: int, i: np.ndarray) -> np.ndarray:
    """splitmix64's finaliser of x + (i + 1) * golden, vectorised over i."""
    i = np.asarray(i, np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(x & _M64) + (i + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def stream_uniforms(seed: int, stream: int, n: int) -> np.ndarray:
    """Row i's uniform of stream k: the top 53 bits of splitmix(splitmix(seed, k), i) over 2^53."""
    key = int(splitmix(seed, np.array([stream], np.uint64))[0])
    return (splitmix(key, np.arange(n, dtype=np.uint64)) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def split_bounds(weights: Sequence[float]) -> List[float]:
    w = [float(x) for x in weights]
    total = sum(w)
    b = [0.0]
    for x in w:
        b.append(b[-1] + x / total)
    return b


def sample_rows(n: int, seed: int, fraction: float) -> np.ndarray:
    """Dataset.sample(fraction) (BernoulliCellSampler): row i is kept when its stream-0 uniform is < fraction."""
    return np.flatnonzero(stream_uniforms(seed, 0, n) < fraction)


def split_samples(n: int, seed: int, fraction: float = 0.1, weights=(0.8, 0.2)) -> List[np.ndarray]:
    """sample(fraction), then randomSplit(weights) of the sampled rows: a sampled row i goes to part j when
    lb_j <= u_i < ub_j, u_i its stream-1 uniform.  Row indices ascending per part."""
    rows = sample_rows(n, seed, fraction)
    u = stream_uniforms(seed, 1, n)[rows]
    b = split_bounds(weights)
    return [rows[(u >= lo) & (u < hi)] for lo, hi in zip(b[:-1], b[1:])]


def split_samples_by_timestamp(timestamp, seed: int, fraction: float = 0.1, relative_error: float = 0.05):
    """sample(fraction), then approxQuantile(timestamp, 0.8, relative_error) of the sampled rows as one summary:
    rows with timestamp <= it train, the rest test.  Returns (train rows, test rows, split timestamp)."""
    ts = np.asarray(timestamp, np.int64)
    rows = sample_rows(len(ts), seed, fraction)
    if rows.size == 0:
        return rows, rows, math.nan
    split = float(one_summary_quantiles(ts[rows].astype(np.float64), [0.8], relative_error)[0])
    t = ts[rows].astype(np.float64)
    return rows[t <= split], rows[t > split], split
