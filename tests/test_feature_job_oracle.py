"""The FeatureEngineering job's oracle (`oracle/feature_job.py`) on the CPU: hand-worked known answers for Spark's
QuantileSummaries, the discretizer, the scaler, the Scala 2.11 hash-trie order and the encoders, the whole-file
rating features of the fixture, and the sample / split draws."""
import math
import os

import numpy as np
import pytest

from oracle import feature_job as J
from oracle.feature_eng import java_string_hash

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
REF_DATA = "/root/reference/src/main/resources/webroot/sampledata"


def _movies():
    return np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))


# -------------------------------------------------------------------------------------------- QuantileSummaries
def test_ten_values_known_answers():
    # 1..10, eps 0.1: deltas floor(0.2 (i + 1)) = 0,0,0,0,1,1,1,1,1 and 0 at the end; T = 2, so nothing merges.
    _, s, n = J.one_summary_samples(np.arange(1, 11), 0.1)
    assert n == 10 and s == [[float(v), 1, d] for v, d in zip(range(1, 11), [0, 0, 0, 0, 1, 1, 1, 1, 1, 0])]
    q = J.one_summary_quantiles(np.arange(1, 11), [0.0, 0.05, 0.1, 0.11, 0.5, 0.9, 0.95, 1.0], 0.1)
    # p <= eps -> min; p >= 1 - eps (0.9) -> max; 0.11: rank 2, targetError 1, minRank 1 of value 1 already fits;
    # 0.5: rank 5, the first sample with minRank + 1 >= 5 is value 4
    assert q.tolist() == [1, 1, 1, 1, 4, 10, 10, 10]


def test_target_error_rule():
    # 10..50, eps 0.15: rank(0.5) = 3, deltas 0,0,0,1,0.  ceil(0.75) = 1 picks 20 (minRank 2 + 1 >= 3); the
    # unrounded 0.75 needs minRank >= 2.25 and picks 30.
    v = [10, 20, 30, 40, 50]
    assert J.one_summary_quantiles(v, [0.5], 0.15).tolist() == [20]
    assert J.one_summary_quantiles(v, [0.5], 0.15, target_error_ceil=False).tolist() == [30]


def test_duplicates():
    # four 1s and a 5: every quantile between the ends is a 1
    q = J.one_summary_quantiles([1, 5, 1, 1, 1], [0.25, 0.5, 0.75, 1.0], 0.001)
    assert q.tolist() == [1, 1, 1, 5]


def test_compress_on_both_sides_of_one_over_two_eps():
    # eps 0.01: n = 99 gives T = 1.98 < 2, every sample survives; n = 101 gives T = 2.02, so a head of delta 0
    # absorbs one sample: 100 takes 99, 98..49 (delta 1) stay alone, 48 takes 47, ..., 2 takes 1; plus the minimum.
    _, s, _ = J.one_summary_samples(np.arange(99), 0.01)
    assert len(s) == 99 and all(g == 1 for _, g, _ in s)
    _, s, _ = J.one_summary_samples(np.arange(101), 0.01)
    assert len(s) == 1 + 50 + 24 + 1 and sum(g for _, g, _ in s) == 101
    assert s[-1] == [100.0, 2, 0] and s[0] == [0.0, 1, 0] and s[1] == [2.0, 2, 0] and s[25] == [49.0, 1, 1]


@pytest.mark.parametrize("eps", [0.0, 0.001, 0.01, 0.05, 0.3, 1.0])
def test_closed_form_is_the_literal_compress(eps):
    for n in list(range(1, 40)) + [99, 100, 101, 499, 500, 501, 999, 1000, 1001, 4567]:
        _, s, _ = J.one_summary_samples(np.arange(n), eps)
        assert [(int(v), g, d) for v, g, d in s] == J.one_summary_closed_form(n, eps), n


@pytest.mark.parametrize("eps", [0.0, 1e-5, 0.0004, 0.001, 0.00101, 0.01, 0.05, 0.3, 1.0])
def test_segment_walk_is_the_literal_compress(eps):
    """The device's walk, one step per run of equal delta, on sizes where 2 eps n falls below, at and just above 2
    (long runs whose heads absorb one sample each) and far above it."""
    for n in list(range(1, 30)) + [999, 1000, 1001, 1500, 2001, 4567, 10001, 100000, 200001]:
        _, s, _ = J.one_summary_samples(np.arange(n), eps)
        assert [(int(v), g, d) for v, g, d in s] == J.one_summary_segments(n, eps), (n, eps)


def test_one_value_and_both_ends():
    assert J.one_summary_quantiles([7.5], [0, 0.3, 1], 0.001).tolist() == [7.5] * 3
    # p 0.5 of three values: rank 2, targetError ceil(0.003) = 1, and the minimum's minRank 1 already fits
    q = J.one_summary_quantiles([-np.inf, 3, np.inf], [0, 0.5, 0.67, 1], 0.001)
    assert q.tolist() == [-np.inf, -np.inf, 3, np.inf]
    with pytest.raises(ValueError):
        J.one_summary_quantiles([1, np.nan], [0.5], 0.01)


def test_partitions_below_1000_values_give_the_one_summary_answer():
    """Up to 999 values (eps 0.001) spread over 200 partitions: per-partition deltas are 0 and no merge passes
    2 eps n < 2, so any split into partitions answers as one summary does - with targetError = ceil(eps n) only."""
    rng = np.random.default_rng(1)
    probs = [k / 100 for k in range(101)]
    differs_unrounded = 0
    for n in (1, 2, 17, 499, 500, 731, 999):
        v = rng.integers(1, 400, n).astype(np.float64)
        asg = rng.integers(0, 200, n)
        parts = [v[asg == k].tolist() for k in range(200) if (asg == k).any()]
        assert J.spark_approx_quantile(parts, probs, 0.001) == J.one_summary_quantiles(v, probs, 0.001).tolist()
        differs_unrounded += J.spark_approx_quantile(parts, probs, 0.001, target_error_ceil=False) != \
            J.one_summary_quantiles(v, probs, 0.001, target_error_ceil=False).tolist()
    assert differs_unrounded > 0


def test_above_the_bounds_the_answers_part():
    rng = np.random.default_rng(2)
    probs = [k / 100 for k in range(101)]
    v = rng.integers(1, 5000, 20000).astype(np.float64)
    asg = rng.integers(0, 8, v.size)
    parts = [v[asg == k].tolist() for k in range(8)]
    assert J.spark_approx_quantile(parts, probs, 0.001) != J.one_summary_quantiles(v, probs, 0.001).tolist()
    # one partition: equal below the 50 000-value head buffer, not above it (the buffer is flushed and compressed)
    for n, same in ((49999, True), (60000, False)):
        w = rng.permutation(n).astype(np.float64)
        assert (J.spark_approx_quantile([w.tolist()], probs, 0.01) ==
                J.one_summary_quantiles(w, probs, 0.01).tolist()) == same, n


# ------------------------------------------------------------------------------ discretizer, bucketizer, scaler
def test_duplicate_splits_leave_fewer_buckets():
    s = J.discretizer_splits([1, 5, 1, 1, 1], 4)
    assert s.tolist() == [-np.inf, 1, np.inf]
    assert J.bucketize(s, [1, 5, 0.5, 1]).tolist() == [1, 1, 0, 1]


def test_discretizer_probabilities_are_the_scala_range():
    # 1 / 11 prints as 0.09090909090909091 > 1/11: BigDecimal 1 quot it is 10, so 11 elements, ending at 10 step
    p = J.discretizer_probabilities(11)
    assert len(p) == 11 and p[-1] == 10 * (1 / 11) == 0.9090909090909092
    # 0.01 is exactly 1/100: 101 elements, element k = 0.01 * k, which is not always k / 100
    p = J.discretizer_probabilities(100)
    assert len(p) == 101 and p[-1] == 1.0 and p[57] == 0.01 * 57 != 0.57
    assert J.discretizer_probabilities(2) == [0.0, 0.5, 1.0]
    assert len(J.discretizer_probabilities(13)) == 13
    # eleven buckets of 0..109: the 10/11 quantile is lost to the +inf end, ten buckets remain
    s = J.discretizer_splits(np.arange(110.0), 11)
    assert len(s) == 11 and s[-1] == np.inf and s[-2] < 100


def test_bucketizer_edges():
    s = [-np.inf, 0, 10, np.inf]
    assert J.bucketize(s, [-np.inf, -1, 0, 5, 10, np.inf]).tolist() == [0, 0, 1, 1, 2, 2]
    assert J.bucketize([0, 1, 2], [0, 1, 1.5, 2]).tolist() == [0, 1, 1, 1]       # the last bucket includes 2
    for bad in ([np.nan], [3], [-1]):
        with pytest.raises(ValueError):
            J.bucketize([0, 1, 2], bad)
    with pytest.raises(ValueError):
        J.discretizer_splits([np.inf, np.inf], 2)                                    # splits -inf, inf: one bucket


def test_min_max_scaler():
    assert J.min_max_scale([3.0, 3.0, 3.0])[0].tolist() == [0.5] * 3
    out, lo, hi = J.min_max_scale([2.0, 1.0, 4.0])
    assert (lo, hi) == (1.0, 4.0) and out.tolist() == [1 / 3, 0.0, 1.0]
    with pytest.raises(ValueError):
        J.min_max_scale([1.0, np.nan])


# ---------------------------------------------------------------------------------------- the Scala 2.11 trie
def test_improve_by_hand():
    # "a".hashCode = 97; h = 97 + ~(97 << 9) = 0xFFFF3E60; h ^= h >>> 14 -> 0xFFFCC19C; h += h << 4 -> 0xFFC8DB5C;
    # h ^ (h >>> 10) = 0xFFF7296A, whose low 5 bits are 10
    assert J.improve(97) == 0xFFF7296A
    # level-0 digits: e 0, f 8, a 10, b 18, c 25, d 31 - no two share one, so the trie iterates in that order
    assert [J.improve(java_string_hash(w)) & 31 for w in "abcdef"] == [10, 18, 25, 31, 0, 8]
    assert J.hash_trie_keys(list("abcdef")) == list("efabcd")
    assert J.hash_trie_keys(list("fedcba")) == list("efabcd")


def test_trie_closed_form_on_the_genre_words():
    m = _movies()
    words = sorted({w for g in m["genres"] for w in g.split("|")}) + ["(no genres listed)"]
    assert len(words) == 20
    by_key = sorted(words, key=lambda w: J.trie_order_key(java_string_hash(w)))
    assert J.hash_trie_keys(words) == by_key
    assert J.hash_trie_keys(words[::-1]) == by_key


def test_genre_labels_of_movies_csv():
    m = _movies()
    labels, counts = J.string_indexer_labels([w for g in m["genres"] for w in g.split("|")])
    assert len(labels) == 19 and counts == sorted(counts, reverse=True)
    # the two ties of the reference's movies.csv, in trie order
    assert labels[8:10] == ["Mystery", "Sci-Fi"] and counts[8:10] == [51, 51]
    assert labels[12:14] == ["War", "Documentary"] and counts[12:14] == [34, 34]


def test_one_hot_and_multi_hot():
    idx, size = J.one_hot([3, 1, 7])
    assert idx.tolist() == [3, 1, 7] and size == 8
    labels, counts, ids, off, ind = J.multi_hot([1, 3, 2], ["A|B", "B", "C|A|B"])
    assert labels == ["B", "A", "C"] and counts == [3, 2, 1]
    assert ids.tolist() == [1, 2, 3] and off.tolist() == [0, 2, 5, 6] and ind.tolist() == [0, 1, 0, 1, 2, 0]
    with pytest.raises(ValueError):
        J.multi_hot([1], ["A|A"])


# --------------------------------------------------------------------------------------------- rating features
def test_rating_features_by_hand():
    # movie 2: 4.0, 3.0 -> avg 3.5, var 0.5; movie 5: one 2.5 -> var null; movie 9: 5, 5, 4 -> avg 14/3, var 1/3
    ids, n, avg, var = J.rating_features([2, 5, 2, 9, 9, 9], [8, 5, 6, 10, 10, 8])
    assert ids.tolist() == [2, 5, 9] and n.tolist() == [2, 1, 3]
    assert avg.tolist() == [3.5, 2.5, 14 / 3] and var[0] == 0.5 and math.isnan(var[1]) and var[2] == 1 / 3


def test_whole_file_rating_features_from_the_fixture_moments():
    m = _movies()
    ids, n, avg, var = J.rating_features_from_moments(m["all_count"], m["all_sum_half"], m["all_sum_half2"])
    assert len(ids) == 981 and np.isnan(var).sum() == np.count_nonzero(n == 1)
    ok = n > 1
    mean = m["all_sum_half"][ids] / 2.0 / n
    assert np.allclose(avg, mean, rtol=1e-15, atol=0)
    e2 = m["all_sum_half2"][ids][ok] / 4.0 / n[ok]
    assert np.allclose(var[ok], (e2 - mean[ok] ** 2) * n[ok] / (n[ok] - 1), rtol=1e-9, atol=1e-12)
    splits = J.discretizer_splits(n.astype(np.float64), 100)
    # 981 movies in 200 partitions answer as one summary does
    rng = np.random.default_rng(3)
    asg = rng.integers(0, 200, n.size)
    parts = [n[asg == k].astype(np.float64).tolist() for k in range(200) if (asg == k).any()]
    q = J.spark_approx_quantile(parts, J.discretizer_probabilities(100), 0.001)
    q[0], q[-1] = -np.inf, np.inf
    assert list(dict.fromkeys(q)) == splits.tolist()
    b = J.bucketize(splits, n.astype(np.float64))
    assert b.min() == 0 and b.max() == len(splits) - 2
    scaled = J.min_max_scale(avg)[0]
    assert scaled.min() == 0.0 and scaled.max() == 1.0


# ----------------------------------------------------------------------------------------------- sample, split
def test_split_of_a_million_uniforms_is_within_five_sigma():
    n = 1000000
    train, test = J.split_samples(n, seed=11, fraction=1.0)
    assert train.size + test.size == n and abs(train.size - 0.8 * n) < 5 * math.sqrt(n * 0.8 * 0.2)
    sampled = J.sample_rows(n, seed=11, fraction=0.1)
    assert abs(sampled.size - 0.1 * n) < 5 * math.sqrt(n * 0.1 * 0.9)


def test_weights_do_not_change_the_sample():
    a = J.split_samples(10000, seed=5, weights=(0.8, 0.2))
    b = J.split_samples(10000, seed=5, weights=(1, 1, 1))
    assert np.array_equal(np.sort(np.concatenate(a)), np.sort(np.concatenate(b)))


def test_timestamp_split_orders_the_parts():
    rng = np.random.default_rng(4)
    ts = rng.integers(800000000, 1600000000, 50000)
    train, test, split = J.split_samples_by_timestamp(ts, seed=9)
    assert train.size and test.size and ts[train].max() <= split < ts[test].min()
    assert abs(train.size / (train.size + test.size) - 0.8) < 0.05


@pytest.mark.skipif(not os.path.isdir(REF_DATA), reason="the reference's sample data is not here")
def test_fixtures_are_the_reference_csvs():
    import csv
    m = _movies()
    with open(os.path.join(REF_DATA, "movies.csv"), newline="", encoding="utf-8") as f:
        rows = list(csv.reader(f))[1:]
    assert [int(r[0]) for r in rows] == m["movieId"].tolist() and [r[2] for r in rows] == m["genres"].tolist()
    a = np.loadtxt(os.path.join(REF_DATA, "ratings.csv"), delimiter=",", skiprows=1)
    mid, half = a[:, 1].astype(np.int64), (a[:, 2] * 2).astype(np.int64)
    slots = len(m["all_count"])
    assert np.array_equal(np.bincount(mid, minlength=slots), m["all_count"])
    assert np.array_equal(np.bincount(mid, half, slots).astype(np.int64), m["all_sum_half"])
    assert np.array_equal(np.bincount(mid, half * half, slots).astype(np.int64), m["all_sum_half2"])
