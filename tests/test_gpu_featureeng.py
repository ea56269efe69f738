"""The sample builder on the device (`featureeng.build_samples`, csrc/featureeng.cu) against the numpy oracle."""

import numpy as np
import pytest

from oracle import feature_eng as F
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import featureeng as FE
from sparrowrecsys_b200.model import launch_count

from test_featureeng_oracle import (MOVIE_STAT_COLS, TIE_FREE, all_movie_features, check_hand, fixture_inputs,
                                    hand_inputs, model_samples, tie_classes)

pytestmark = pytest.mark.gpu


def _bit_equal(a, b):
    assert set(a) == set(b) == set(F.COLUMNS)
    for c in F.COLUMNS:
        x, y = a[c], b[c]
        assert x.dtype == y.dtype and x.shape == y.shape, (c, x.dtype, y.dtype, x.shape, y.shape)
        if x.dtype == np.float32:
            x, y = x.view(np.int32), y.view(np.int32)
        bad = np.flatnonzero(x != y)
        assert bad.size == 0, (c, bad[:5], x[bad[:5]], y[bad[:5]])


@pytest.fixture(scope="module")
def full():
    ratings, movies = fixture_inputs()
    dev = FE.build_samples(ratings, movies, device=0)
    return ratings, movies, dev


def test_full_fixture_bit_for_bit_against_the_oracle(full):
    ratings, movies, dev = full
    _bit_equal(dev, F.build_samples(ratings, movies))
    assert len(dev["movieId"]) == 193207


def test_two_runs_give_the_same_bits(full):
    ratings, movies, dev = full
    _bit_equal(dev, FE.build_samples(ratings, movies, device=0))


def test_hand_built_known_answers_on_the_device():
    ratings, movies = hand_inputs()
    dev = FE.build_samples(ratings, movies, device=0)
    check_hand(dev)
    _bit_equal(dev, F.build_samples(ratings, movies))


def _raw_call(user, movie, half, ts, year, genres, n_genres=1, hashes=None):
    import ctypes as C
    n = len(user)
    bufs = {f: np.zeros(max(n, 1) * 5, np.int32) for f, _ in _lib.SrsSamples._fields_}
    st = _lib.SrsSamples(**{k: v.ctypes.data for k, v in bufs.items()})
    hashes = np.zeros(max(n_genres, 1), np.int32) if hashes is None else hashes
    kept = C.c_int64(-1)
    a = [np.ascontiguousarray(x, t) for x, t in ((user, np.int32), (movie, np.int32), (half, np.int8),
                                                 (ts, np.int32), (year, np.int32), (genres, np.int32))]
    rc = _lib.load().srs_featureeng_host(*[x.ctypes.data for x in a[:4]], n, a[4].ctypes.data, a[5].ctypes.data,
                                         a[4].shape[0], a[5].shape[1], hashes.ctypes.data, n_genres, 0,
                                         C.byref(st), C.byref(kept))
    return rc, kept.value


def test_rejections_leave_no_launch_behind():
    u = np.array([1, 1, 1])
    m = np.array([1, 2, 1])
    h = np.array([8, 7, 10])
    t = np.array([5, 6, 7])
    year = np.full(3, 1990)
    genres = np.array([[-1], [0], [-1]])
    rc, kept = _raw_call(u, m, h, t, year, genres)
    assert rc == _lib.SRS_OK and kept == 1
    n0 = launch_count()
    for args in ((u, m, np.array([8, 0, 10]), t, year, genres),           # rating 0: not a half-star in [0.5, 5]
                 (u, m, np.array([8, 11, 10]), t, year, genres),          # 5.5
                 (np.array([1, -1, 1]), m, h, t, year, genres),           # negative user id
                 (u, np.array([1, -2, 1]), h, t, year, genres),           # negative movie id
                 (u, np.array([1, 3, 1]), h, t, year, genres),            # movie outside the table
                 (u, m, h, np.array([5, 0, 7]), year, genres),            # timestamp not positive
                 (u, m, h, np.array([5, -6, 7]), year, genres),
                 (u, m, h, t, year, np.array([[-1], [1], [-1]])),         # genre index past the vocabulary
                 (u, m, h, t, np.array([1990, 10000, 1990]), genres)):    # not a four-character year
        rc, kept = _raw_call(*args)
        assert rc == _lib.SRS_ERR_INVALID and kept == 0, args
    assert launch_count() == n0
    with pytest.raises(ValueError):
        FE.build_samples({"userId": u, "movieId": m, "rating": np.array([4.0, 3.3, 5.0]), "timestamp": t},
                         {"movieId": np.array([1]), "title": ["A (1999)"], "genres": ["Drama"]})
    assert launch_count() == n0


def test_write_samples_csv_reproduces_the_tie_free_model_samples_text(full, tmp_path):
    ratings, movies, dev = full
    ms, text = model_samples()
    n = len(text) - 1
    cls, _, _, back = tie_classes(ratings)
    key = lambda u, m: np.asarray(u, np.int64) * 100000 + np.asarray(m, np.int64)
    kf = key(ratings["userId"], ratings["movieId"])
    sf = np.argsort(kf)
    fr = sf[np.searchsorted(kf[sf], key(ms["userId"][:n], ms["movieId"][:n]))]
    tf = np.flatnonzero(cls[fr] == TIE_FREE)
    assert len(tf) > 500
    kd = key(dev["userId"], dev["movieId"])
    sd = np.argsort(kd)
    rows = sd[np.searchsorted(kd[sd], key(ms["userId"][tf], ms["movieId"][tf]))]
    got = {c: v[rows] for c, v in dev.items()}
    # the fixture holds a subset of the users, so the movie columns, which span every user, are the ones the
    # movies' rating moments over the whole of ratings.csv give (pinned in test_featureeng_oracle.py)
    for c, v in zip(MOVIE_STAT_COLS, all_movie_features()):
        got[c] = v[got["movieId"]]
    path = tmp_path / "samples.csv"
    FE.write_samples_csv(str(path), got)
    lines = path.read_text().splitlines(keepends=True)
    want = [text[0]] + [text[1 + r] for r in tf.tolist()]
    assert lines == [t.replace("\r\n", "\n") for t in want]


@pytest.mark.parametrize("model", ["neuralcf", "deepfm"])
def test_fit_on_built_samples_matches_fit_on_csv_text(full, tmp_path, model):
    """One epoch on a slice of the built rows gives the bits of one epoch on the same rows read back from CSV."""
    from sparrowrecsys_b200.features import load_samples_csv
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.training import Trainer
    from sparrowrecsys_b200.weights import init_weights
    _, _, dev = full
    part = {c: v[:3000] for c, v in dev.items()}
    path = tmp_path / "part.csv"
    FE.write_samples_csv(str(path), part)
    text = load_samples_csv(str(path))
    spec = default_spec(model)
    W0 = init_weights(spec, 3, for_test=False)
    runs = []
    for feats in (part, text):
        with Trainer(spec, W0, device=0) as tr:
            hist = tr.fit(feats, epochs=1, batch_size=64, seed=0)
            runs.append((hist, tr.weights()))
    (h1, w1), (h2, w2) = runs
    assert h1 == h2
    for k in w1:
        assert np.array_equal(w1[k], w2[k]), k
