"""The FeatureEngineering job and the sample / split on the device (`featurejob.py`, csrc/featurejob.cu) against the
numpy oracle (`oracle/feature_job.py`), bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import feature_job as J
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import featureeng as FE
from sparrowrecsys_b200 import featurejob as FJ
from sparrowrecsys_b200.model import launch_count

from test_featureeng_oracle import fixture_inputs

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    if a.dtype.kind == "f":
        a, b = a.view(np.int64 if a.itemsize == 8 else np.int32), b.view(np.int64 if b.itemsize == 8 else np.int32)
    bad = np.flatnonzero(a.reshape(-1) != b.reshape(-1))
    assert bad.size == 0, (bad[:5], a.reshape(-1)[bad[:5]], b.reshape(-1)[bad[:5]])


@pytest.fixture(scope="module")
def fixture():
    return fixture_inputs()


# -------------------------------------------------------------------------------------------------- quantiles
@pytest.mark.parametrize("eps", [0.0, 0.001, 0.01, 0.05, 0.3, 1.0])
def test_approx_quantile_matches_the_one_summary_oracle(eps):
    rng = np.random.default_rng(7)
    probs = np.array([0, eps, eps * 1.5, 0.1, 0.25, 0.5, 0.8, 0.999, 1 - eps, 1.0]).clip(0, 1)
    for n in (1, 2, 3, 10, 99, 101, 999, 1000, 4567, 60001):
        v = rng.integers(-50, 300, n).astype(np.float64) * 0.5        # many duplicates
        if n > 3:
            v[:3] = [-np.inf, np.inf, -0.0]
        got = FJ.approx_quantile(v, probs, eps)
        _same_bits(got, J.one_summary_quantiles(v, probs, eps))


@pytest.mark.parametrize("n,eps", [(1001, 0.001), (1500, 0.001), (3001, 0.001), (200001, 1e-5), (150001, 2e-5),
                                   (100000, 1e-5), (120000, 0.0001)])
def test_approx_quantile_where_few_samples_merge(n, eps):
    """2 eps n just above 2 (heads absorb one sample in long runs) and eps near 1 / n: the segment walk and the
    binary-search query against the literal compress and query."""
    rng = np.random.default_rng(n)
    v = rng.normal(size=n)
    probs = np.r_[0.0, eps, np.linspace(0.001, 0.999, 97), 1 - eps, 1.0]
    _same_bits(FJ.approx_quantile(v, probs, eps), J.one_summary_quantiles(v, probs, eps))


def test_hand_worked_quantiles_on_the_device():
    assert FJ.approx_quantile(np.arange(1, 11), [0.0, 0.05, 0.11, 0.5, 0.9, 1.0], 0.1).tolist() == [1, 1, 1, 4, 10, 10]
    assert FJ.approx_quantile([10, 20, 30, 40, 50], [0.5], 0.15).tolist() == [20]       # targetError = ceil(eps n)
    assert FJ.approx_quantile([7.5], [0, 0.5, 1], 0.001).tolist() == [7.5] * 3


@pytest.mark.parametrize("num_buckets", [2, 11, 13, 100, 1000])
def test_discretizer_on_the_fixture_counts(num_buckets):
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    _, n, _, _ = J.rating_features_from_moments(m["all_count"], m["all_sum_half"], m["all_sum_half2"])
    x = n.astype(np.float64)
    bz, b = FJ.QuantileDiscretizer(num_buckets).fit_transform(x)
    want = J.discretizer_splits(x, num_buckets)
    _same_bits(bz.splits, want)
    _same_bits(b, J.bucketize(want, x))
    _same_bits(FJ.QuantileDiscretizer(num_buckets).fit(x).transform(x), b)


def test_discretizer_edges():
    bz = FJ.QuantileDiscretizer(11).fit(np.arange(110.0))                         # a range of 11 elements
    _same_bits(bz.splits, J.discretizer_splits(np.arange(110.0), 11))
    assert len(bz.splits) == 11
    bz, b = FJ.QuantileDiscretizer(4).fit_transform([1, 5, 1, 1, 1])
    assert bz.splits.tolist() == [-np.inf, 1, np.inf] and b.tolist() == [1] * 5
    bz, b = FJ.QuantileDiscretizer(100).fit_transform(np.full(777, 3.0))            # all equal: one bucket used
    assert bz.splits.tolist() == [-np.inf, 3, np.inf] and set(b.tolist()) == {1.0}
    bz, b = FJ.QuantileDiscretizer(10).fit_transform([42.0])
    assert bz.splits.tolist() == [-np.inf, 42, np.inf] and b.tolist() == [1.0]
    bk = FJ.Bucketizer([-np.inf, 0, 10, np.inf])
    assert bk.transform([-np.inf, -1, 0, 5, 10, np.inf]).tolist() == [0, 0, 1, 1, 2, 2]
    assert FJ.Bucketizer([0, 1, 2]).transform([0, 1, 1.5, 2]).tolist() == [0, 1, 1, 1]
    with pytest.raises(_lib.SrsInvalidError):
        FJ.QuantileDiscretizer(2).fit([np.inf, np.inf])                               # splits -inf, +inf


def test_min_max_scaler(fixture):
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    _, _, avg, _ = J.rating_features_from_moments(m["all_count"], m["all_sum_half"], m["all_sum_half2"])
    model, out = FJ.MinMaxScaler().fit_transform(avg)
    want, lo, hi = J.min_max_scale(avg)
    _same_bits(out, want)
    assert (model.original_min, model.original_max) == (lo, hi)
    _same_bits(model.transform(avg[::-1]), want[::-1])
    assert FJ.MinMaxScaler().fit_transform([3.0, 3.0])[1].tolist() == [0.5, 0.5]


# ----------------------------------------------------------------------------------------- the job's results
def test_rating_features_on_the_fixture(fixture):
    ratings, _ = fixture
    got = FJ.rating_features(ratings)
    ids, n, avg, var = J.rating_features(ratings["movieId"], (ratings["rating"] * 2).astype(np.int64))
    _same_bits(got["movieId"], ids)
    _same_bits(got["ratingCount"], n)
    _same_bits(got["avgRating"], avg)
    _same_bits(got["ratingVar"], var)


def test_rating_features_at_the_largest_movie_id():
    r = {"movieId": np.array([2 ** 24 - 1, 0, 2 ** 24 - 1]), "rating": np.array([4.5, 1.0, 2.0])}
    got = FJ.rating_features(r)
    assert got["movieId"].tolist() == [0, 2 ** 24 - 1] and got["ratingCount"].tolist() == [1, 2]
    assert got["avgRating"].tolist() == [1.0, 3.25] and np.isnan(got["ratingVar"][0])
    assert got["ratingVar"][1] == 3.125


def test_string_indexer_and_multi_hot_on_movies_csv(fixture):
    _, movies = fixture
    mh = FJ.multi_hot(movies["movieId"], movies["genres"])
    labels, counts, ids, off, ind = J.multi_hot(movies["movieId"], movies["genres"])
    assert mh["labels"] == labels and mh["counts"].tolist() == counts and mh["size"] == 19
    _same_bits(mh["movieId"], ids)
    _same_bits(mh["offsets"], off.astype(np.int32))
    _same_bits(mh["indices"], ind)
    model = FJ.StringIndexer().fit([w for g in movies["genres"] for w in g.split("|")] + ["(no genres listed)"])
    assert model.labels[-1] == "(no genres listed)" and model.labels[:19] == labels


def test_multi_hot_by_hand():
    mh = FJ.multi_hot([1, 3, 2], ["A|B", "B", "C|A|B"])
    assert mh["labels"] == ["B", "A", "C"] and mh["movieId"].tolist() == [1, 2, 3]
    assert mh["offsets"].tolist() == [0, 2, 5, 6] and mh["indices"].tolist() == [0, 1, 0, 1, 2, 0]
    assert FJ.StringIndexer().fit(list("abcdefab")).labels == list("abefcd")            # a, b twice; then trie order


def test_feature_engineering_on_the_fixture(fixture):
    ratings, movies = fixture
    r = FE.feature_engineering(ratings, movies)
    ids, n, avg, var, bucket, scaled, splits = J.feature_engineering(ratings["movieId"],
                                                                     (ratings["rating"] * 2).astype(np.int64))
    mf = r["movie_features"]
    for k, want in (("movieId", ids), ("ratingCount", n), ("avgRating", avg), ("ratingVar", var),
                    ("ratingCountBucket", bucket), ("scaleAvgRating", scaled), ("splits", splits)):
        _same_bits(mf[k], want)
    assert r["one_hot"]["size"] == int(movies["movieId"].max()) + 1
    assert r["multi_hot"]["size"] == 19


def test_same_bits_twice_and_rejections_launch_nothing(fixture):
    ratings, movies = fixture
    a, b = FE.feature_engineering(ratings, movies), FE.feature_engineering(ratings, movies)
    for k in a["movie_features"]:
        _same_bits(a["movie_features"][k], b["movie_features"][k])
    lib = _lib.load()
    p = lambda x: x.ctypes.data
    n0 = launch_count()
    out = np.full(4, 123.0)
    for v, probs, eps in (([1.0, np.nan], [0.5], 0.01), ([1.0], [1.5], 0.01), ([1.0], [0.5], -0.1)):
        v, probs = np.array(v), np.array(probs)
        assert lib.srs_approx_quantile_host(p(v), v.size, p(probs), probs.size, eps, 0, p(out)) == _lib.SRS_ERR_INVALID
    splits = np.array([0.0, 1.0, 2.0])
    b32 = np.full(2, -7, np.int32)
    for v in ([0.5, 3.0], [np.nan, 1.0]):
        v = np.array(v)
        assert lib.srs_bucketize_host(p(splits), 3, p(v), 2, 0, p(b32)) == _lib.SRS_ERR_INVALID
    w = np.array([0.8, -0.2])
    rows, cnt = np.full(4, -7, np.int32), np.full(2, -7, np.int64)
    assert lib.srs_sample_split_host(4, 1, 0.5, p(w), 2, 0, p(rows), p(cnt)) == _lib.SRS_ERR_INVALID
    with pytest.raises(ValueError):
        FJ.multi_hot([1, 2], ["A|A", "B"])
    with pytest.raises(ValueError):
        FJ.rating_features({"movieId": np.array([1]), "rating": np.array([3.3])})
    with pytest.raises(ValueError):
        FJ.MinMaxScaler().fit([np.nan])
    assert launch_count() == n0
    assert (out == 123.0).all() and (b32 == -7).all() and (rows == -7).all() and (cnt == -7).all()


# ----------------------------------------------------------------------------------------------- sample, split
def _check_parts(parts, sampled):
    allr = np.concatenate(parts)
    assert np.unique(allr).size == allr.size                                    # disjoint
    assert np.array_equal(np.sort(allr), sampled)                               # cover the sampled rows
    for p in parts:
        assert np.all(np.diff(p) > 0)                                           # input order


def test_split_rows_match_the_oracle():
    for n, seed, frac, w in ((1, 0, 1.0, (0.8, 0.2)), (1000, 3, 0.1, (0.8, 0.2)), (100000, 2 ** 64 - 1, 0.3, (1, 2, 3)),
                             (250000, 42, 1.0, (0.8, 0.2))):
        got = FJ.sample_split_rows(n, seed, frac, w)
        want = J.split_samples(n, seed, frac, w)
        assert len(got) == len(want)
        for g, x in zip(got, want):
            assert np.array_equal(g, x)
        _check_parts(got, J.sample_rows(n, seed, frac))


def test_timestamp_split(fixture):
    ratings, _ = fixture
    ts = ratings["timestamp"]
    tr, te, split = FJ.sample_split_rows_by_timestamp(ts, 5)
    wtr, wte, wsplit = J.split_samples_by_timestamp(ts, 5)
    assert np.array_equal(tr, wtr) and np.array_equal(te, wte) and split == wsplit
    _check_parts([tr, te], J.sample_rows(len(ts), 5, 0.1))
    assert ts[tr].max() <= split < ts[te].min()
    tr, te, split = FJ.sample_split_rows_by_timestamp(ts[:3], 5, fraction=0.0)
    assert tr.size == te.size == 0 and np.isnan(split)


def test_ml20m_sized_input():
    """20 M ratings over 27 278 movies: rating features and the whole discretizer against the oracle, the split
    against the oracle's draws, the timestamp split's quantile against the oracle on the sampled rows."""
    rng = np.random.default_rng(20)
    n, n_movies = 20000263, 27278
    movie = (rng.zipf(1.3, n) % n_movies).astype(np.int32)
    half = rng.integers(1, 11, n).astype(np.int8)
    ratings = {"movieId": movie, "rating": half / 2.0}
    got = FJ.rating_features(ratings)
    ids, cnt, avg, var = J.rating_features(movie, half.astype(np.int64))
    for k, want in (("movieId", ids), ("ratingCount", cnt), ("avgRating", avg), ("ratingVar", var)):
        _same_bits(got[k], want)
    x = cnt.astype(np.float64)
    bz, b = FJ.QuantileDiscretizer(100).fit_transform(x)
    _same_bits(bz.splits, J.discretizer_splits(x, 100))
    _same_bits(b, J.bucketize(bz.splits, x))
    parts = FJ.sample_split_rows(n, 9)
    u0 = J.stream_uniforms(9, 0, n)
    sampled = np.flatnonzero(u0 < 0.1)
    _check_parts(parts, sampled)
    sub = sampled[::997]                                                        # the oracle's split on a subsample
    u1 = J.stream_uniforms(9, 1, n)[sub]
    assert np.array_equal(np.intersect1d(parts[0], sub), sub[u1 < 0.8])
    ts = rng.integers(789652009, 1427784002, n)
    tr, te, split = FJ.sample_split_rows_by_timestamp(ts, 9)
    _check_parts([tr, te], sampled)
    assert split == J.one_summary_quantiles(ts[sampled].astype(np.float64), [0.8], 0.05)[0]
    assert ts[tr].max() <= split < ts[te].min()


def test_end_to_end_build_split_fit_evaluate(fixture, tmp_path):
    """build_samples -> split_samples -> one NeuralCF epoch -> evaluate on the test part; the same as a fit on the
    parts written with write_samples_csv and read back."""
    from sparrowrecsys_b200.features import load_samples_csv
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.training import Trainer
    from sparrowrecsys_b200.weights import init_weights
    ratings, movies = fixture
    samples = FE.build_samples(ratings, movies)
    train, test = FE.split_samples(samples, seed=1)
    assert set(train) == set(samples) and all(train[k].dtype == samples[k].dtype for k in samples)
    assert abs(len(train["movieId"]) / (len(train["movieId"]) + len(test["movieId"])) - 0.8) < 0.02
    texts = []
    for name, part in (("trainingSamples.csv", train), ("testSamples.csv", test)):
        FE.write_samples_csv(str(tmp_path / name), part)
        texts.append(load_samples_csv(str(tmp_path / name)))
    spec = default_spec("neuralcf")
    W0 = init_weights(spec, 3, for_test=False)
    runs = []
    for tr_feats, te_feats in ((train, test), tuple(texts)):
        with Trainer(spec, W0, device=0) as tr:
            hist = tr.fit(tr_feats, epochs=1, batch_size=128, seed=0)
            runs.append((hist, tr.evaluate(te_feats), tr.weights()))
    (h1, e1, w1), (h2, e2, w2) = runs
    assert h1 == h2 and e1 == e2
    for k in w1:
        assert np.array_equal(w1[k], w2[k]), k
