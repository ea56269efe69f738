"""float64 restatement of Spark ML 2.4's BucketedRandomProjectionLSH as the reference's embeddingLSH uses it
(Embedding.scala:230-252): `fit` (java.util.Random Gaussians, normalised), `transform` (bucket ids) and the
single-probe `approxNearestNeighbors`.

THIS IS THE READABLE SPEC, NOT PRODUCT.  Restated from memory of Spark's source and from the algorithm
java.util.Random's javadoc specifies, not from a pinned source; DESIGN.md section 4.14 says which parts are pinned.
Every sum is sequential in double with one rounding per operation (numpy's element-wise float64 operations).
"""
from __future__ import annotations

import math

import numpy as np

_M48 = (1 << 48) - 1
_MULT = 0x5DEECE66D


class JavaRandom:
    """java.util.Random: the 48-bit LCG, nextInt, nextDouble and the polar nextGaussian with its cached second
    value.  StrictMath.log is fdlibm's; math.log here is the C library's, which may differ in the last bit."""

    def __init__(self, seed: int):
        self.state = (seed ^ _MULT) & _M48
        self.have_next = False
        self.next_g = 0.0

    def next_bits(self, bits: int) -> int:
        self.state = (self.state * _MULT + 0xB) & _M48
        v = self.state >> (48 - bits)
        return v - (1 << bits) if v >= 1 << (bits - 1) else v       # Java's int cast

    def next_int(self) -> int:
        return self.next_bits(32)

    def next_double(self) -> float:
        hi = self.next_bits(26) & ((1 << 26) - 1)
        lo = self.next_bits(27) & ((1 << 27) - 1)
        return ((hi << 27) + lo) * 2.0 ** -53

    def next_gaussian(self) -> float:
        if self.have_next:
            self.have_next = False
            return self.next_g
        while True:
            v1 = 2 * self.next_double() - 1
            v2 = 2 * self.next_double() - 1
            s = v1 * v1 + v2 * v2
            if 0 < s < 1:
                break
        m = math.sqrt(-2 * math.log(s) / s)
        self.next_g = v2 * m
        self.have_next = True
        return v1 * m


def java_string_hash(s: str) -> int:
    """String.hashCode: h = 31 h + c over the UTF-16 units, as a signed 32-bit int."""
    h = 0
    for c in s:
        h = (31 * h + ord(c)) & 0xFFFFFFFF
    return h - (1 << 32) if h >= 1 << 31 else h


DEFAULT_SEED = java_string_hash("org.apache.spark.ml.feature.BucketedRandomProjectionLSH")   # HasSeed's default


def fit(dim: int, num_hash_tables: int, seed: int = DEFAULT_SEED) -> np.ndarray:
    """randUnitVectors [num_hash_tables][dim]: per table `dim` nextGaussian draws divided by their L2 norm (the
    squares summed left to right, then sqrt) - breeze's normalize."""
    rand = JavaRandom(seed)
    out = np.zeros((num_hash_tables, dim))
    for j in range(num_hash_tables):
        g = [rand.next_gaussian() for _ in range(dim)]
        sq = 0.0
        for x in g:
            sq = sq + x * x
        norm = math.sqrt(sq)
        out[j] = [x / norm for x in g]
    return out


def _dots(x, uv):
    """x [n][D] float64 against uv [L][D]: [n][L], each summed over d ascending from 0.0."""
    acc = np.zeros((x.shape[0], uv.shape[0]))
    for d in range(x.shape[1]):
        acc = acc + x[:, d:d + 1] * uv[None, :, d]
    return acc


def transform(x, uv, bucket_length):
    """Bucket ids [n][L] float64: floor(dot(x, v_j) / bucketLength), x widened to double."""
    x = np.asarray(x, np.float64).reshape(-1, uv.shape[1])
    return np.floor(_dots(x, uv) / bucket_length)


def approx_nearest_neighbors(ids, x, uv, bucket_length, key, k):
    """Single probe: rows sharing the key's bucket in at least one table, by sqrt(sum (x - key)^2) ascending, ties by
    id then row ascending; the first k.  Returns (ids int32 [<= k], distances float64)."""
    x = np.asarray(x, np.float32).astype(np.float64)
    key = np.asarray(key, np.float64)
    ids = np.asarray(ids, np.int64)
    kh = transform(key[None, :], uv, bucket_length)[0]
    cand = np.flatnonzero(np.any(transform(x, uv, bucket_length) == kh[None, :], axis=1))
    acc = np.zeros(len(cand))
    for d in range(x.shape[1]):
        diff = x[cand, d] - key[d]
        acc = acc + diff * diff
    dist = np.sqrt(acc)
    order = np.lexsort((cand, ids[cand], dist))[:k]
    return ids[cand[order]].astype(np.int32), dist[order]
