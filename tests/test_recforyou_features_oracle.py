"""The "nerualcf" ranker of the Recommended-for-you page with models that read the uf: / mf: features
(oracle/recforyou_features.py, DESIGN.md section 4.26) against hand-built rows, and the rejections of its two C calls
that need no device."""
import numpy as np
import pytest

from oracle import ctr_oracle as O
from oracle import recforyou as R
from oracle.recforyou_features import feature_score_fn, model_movie_id, read_history_keys
from oracle.similar_recall import RecallCatalogue
from sparrowrecsys_b200 import featurestore as FS
from sparrowrecsys_b200.spec import default_spec, history_keys
from sparrowrecsys_b200.weights import init_weights

N_MOVIES, N_USERS = 60, 40
MOVIES = [3, 7, 11, 20, 42]


def _store():
    store = FS.FeatureStore()
    store.backend.hset("uf:5", {"userRatedMovie1": "7", "userRatedMovie2": "11", "userRatedMovie3": "20",
                                "userRatedMovie4": "", "userRatedMovie5": "42", "userGenre1": "Drama",
                                "userGenre2": "Comedy", "userGenre3": "", "userGenre4": "", "userGenre5": "",
                                "userRatingCount": "12", "userAvgRating": "3.75", "userRatingStddev": "0.5"})
    store.backend.hset("uf:6", {"userRatedMovie1": "7", "userRatedMovie2": "9999"})    # past the model
    for i, m in enumerate(MOVIES):
        store.backend.hset("mf:%d" % m, {"movieGenre1": "Action", "movieGenre2": "Drama" if i % 2 else "",
                                         "movieGenre3": "", "movieRatingCount": str(100 + i), "releaseYear": "1995",
                                         "movieAvgRating": "%.2f" % (2.5 + i / 4), "movieRatingStddev": "0.9"})
    return store


def _catalogue():
    ids = list(MOVIES)
    return RecallCatalogue(ids, [["A"]] * len(ids), ids, [5.0, 4.5, 4.0, 3.5, 3.0])


def _rows(user_id, fields, T):
    """The rows of one user over MOVIES, built by hand: history keys by name, the movie side from the table."""
    table = FS.MovieFeatureTable.from_store(_store(), N_MOVIES)
    n = len(MOVIES)
    f = {"movieId": np.array(MOVIES, np.int32), "userId": np.full(n, user_id, np.int32)}
    for k in range(1, T + 1):
        f["userRatedMovie%d" % k] = np.full(n, int(fields.get("userRatedMovie%d" % k, 0)), np.int32)
    for g in range(1, 6):
        col = np.empty(n, dtype=object)
        col[:] = fields.get("userGenre%d" % g, "")
        f["userGenre%d" % g] = col
    f["userRatingCount"] = np.full(n, int(fields.get("userRatingCount", 0)), np.int32)
    f["userAvgReleaseYear"] = np.zeros(n, np.int32)
    f["userReleaseYearStddev"] = np.zeros(n, np.float32)
    f["userAvgRating"] = np.full(n, np.float32(fields.get("userAvgRating", 0.0)), np.float32)
    f["userRatingStddev"] = np.full(n, np.float32(fields.get("userRatingStddev", 0.0)), np.float32)
    f.update(table.gather(np.array(MOVIES)))
    return f


def test_stored_history_keys_land_at_their_ascii_positions():
    keys = history_keys(50)
    assert keys.index("userRatedMovie2") == 11 and keys.index("userRatedMovie5") == 44
    assert keys.index("userRatedMovie1") == 0 and keys.index("userRatedMovie3") == 22
    spec = default_spec("din", emb_dim=8, hist_len=50, n_movies=N_MOVIES, n_users=N_USERS)
    W = init_weights(spec, 3)
    store = _store()
    fn = feature_score_fn(spec, W, store, FS.MovieFeatureTable.from_store(store, N_MOVIES), np.float64)
    # position p of the graph holds history_keys(50)[p]: 11 -> userRatedMovie2 = 11, 44 -> userRatedMovie5 = 42
    by_pos = np.zeros(50, np.int64)
    by_pos[0], by_pos[11], by_pos[22], by_pos[44] = 7, 11, 20, 42
    hand = _rows(5, {"userGenre1": "Drama", "userGenre2": "Comedy", "userRatingCount": 12, "userAvgRating": 3.75,
                     "userRatingStddev": 0.5}, 50)
    for p, k in enumerate(keys):
        hand[k] = np.full(len(MOVIES), by_pos[p], np.int32)
    want = O.forward(spec, W, hand, np.float64)[0].reshape(-1)
    assert fn(5, MOVIES).tobytes() == want.astype(np.float64).tobytes()
    assert read_history_keys(spec) == ["userRatedMovie%d" % k for k in range(1, 6)]
    assert read_history_keys(default_spec("din", hist_len=3)) == ["userRatedMovie1", "userRatedMovie2",
                                                                  "userRatedMovie3"]


@pytest.mark.parametrize("model", ["din", "deepfm", "embeddingmlp", "widendeep"])
def test_a_user_without_a_hash_takes_the_defaults(model):
    spec = default_spec(model, n_movies=N_MOVIES, n_users=N_USERS)
    W = init_weights(spec, 4)
    store = _store()
    assert store.user_features(8) == {}
    fn = feature_score_fn(spec, W, store, FS.MovieFeatureTable.from_store(store, N_MOVIES), np.float64)
    want = O.forward(spec, W, _rows(8, {}, max(spec.hist_len, 5)), np.float64)[0].reshape(-1)
    assert fn(8, MOVIES).tobytes() == want.tobytes()


def test_a_history_id_the_model_reads_decides_model_range():
    store = _store()
    table = FS.MovieFeatureTable.from_store(store, N_MOVIES)
    page = R.RecForYou(_catalogue(), [5, 6, 8])
    for model, want in (("din", R.MODEL_RANGE), ("dien", R.MODEL_RANGE), ("widendeep", R.OK), ("deepfm", R.OK)):
        spec = default_spec(model, n_movies=N_MOVIES, n_users=N_USERS, **({"emb_dim": 8} if model == "dien" else {}))
        fn = feature_score_fn(spec, init_weights(spec, 5), store, table)
        ids, scores, st = page.rec_list(6, 3, "nerualcf", fn)          # userRatedMovie2 = 9999
        assert st == want, model
        assert (len(ids), len(scores)) == ((0, 0) if want == R.MODEL_RANGE else (3, 3))
        assert page.rec_list(5, 3, "nerualcf", fn)[2] == R.OK
        assert page.rec_list(9, 3, "nerualcf", fn)[2] == R.UNKNOWN_USER
    # DIN reads userRatedMovie1..T only: at T = 1 the same user is in range
    spec = default_spec("din", hist_len=1, n_movies=N_MOVIES, n_users=N_USERS)
    assert page.rec_list(6, 3, "nerualcf", feature_score_fn(spec, init_weights(spec, 6), store, table))[2] == R.OK


def test_user_and_candidate_range_rules():
    store = _store()
    spec = default_spec("deepfm", n_movies=N_MOVIES, n_users=6)
    fn = feature_score_fn(spec, init_weights(spec, 7), store, FS.MovieFeatureTable.from_store(store, N_MOVIES))
    page = R.RecForYou(_catalogue(), [5, 6])
    assert page.rec_list(5, 3, "nerualcf", fn)[2] == R.OK
    assert page.rec_list(6, 3, "nerualcf", fn)[2] == R.MODEL_RANGE                # userId 6 == n_users
    small = FS.MovieFeatureTable.from_store(store, 42)                            # candidate 42 past the table
    spec = default_spec("deepfm", n_movies=N_MOVIES, n_users=N_USERS)
    assert page.rec_list(5, 3, "nerualcf", feature_score_fn(spec, init_weights(spec, 7), store, small))[2] == \
        R.MODEL_RANGE
    spec = default_spec("deepfm", n_movies=42, n_users=N_USERS)                   # candidate 42 outside the model
    assert page.rec_list(5, 3, "nerualcf", feature_score_fn(spec, init_weights(spec, 7), store, small))[2] == \
        R.MODEL_RANGE
    # DIN and DIEN check a movie id after float32: 2^24 + 1 reads as 2^24
    din = default_spec("din")
    assert model_movie_id(din, 2 ** 24 + 1) == 2 ** 24 and model_movie_id(spec, 2 ** 24 + 1) == 2 ** 24 + 1
    with pytest.raises(ValueError):
        feature_score_fn(default_spec("neuralcf"), None, store, small)


def _lib():
    from sparrowrecsys_b200 import _lib as L
    return L, L.load()


def test_set_features_rejections_need_no_device():
    L, lib = _lib()
    ids, g, num, hist = (np.zeros(2, np.int32), np.zeros((2, 5), np.int32), np.zeros((2, 3), np.float32),
                         np.zeros((2, 5), np.int32))
    p = lambda a: a.ctypes.data
    assert lib.srs_recforyou_users_set_features_host(None, 2, p(ids), p(g), p(num), p(hist)) == L.SRS_ERR_INVALID
    assert "null user table" in lib.srs_last_error().decode()
    for k in range(4):
        arr = [p(ids), p(g), p(num), p(hist)]
        arr[k] = None
        assert lib.srs_recforyou_users_set_features_host(None, 2, *arr) == L.SRS_ERR_INVALID
        assert "null user_id" in lib.srs_last_error().decode()
    assert lib.srs_recforyou_users_set_features_host(None, -1, p(ids), p(g), p(num), p(hist)) == L.SRS_ERR_INVALID
    assert "< 0" in lib.srs_last_error().decode()


def test_ctr_call_rejections_need_no_device():
    L, lib = _lib()
    q = np.zeros(2, np.int32)
    out = [np.zeros(20, np.int32), np.zeros(20, np.float64), np.zeros(2, np.int32), np.zeros(2, np.int32)]
    p = lambda a: a.ctypes.data
    assert lib.srs_recforyou_ctr_host(None, None, None, p(q), 2, 10, *map(p, out)) == L.SRS_ERR_INVALID
    assert "null model" in lib.srs_last_error().decode()
    for k in range(5):
        arr = [p(q)] + [p(a) for a in out]
        arr[k] = None
        assert lib.srs_recforyou_ctr_host(None, None, None, arr[0], 2, 10, *arr[1:]) == L.SRS_ERR_INVALID
        assert "null user or output array" in lib.srs_last_error().decode()
    for n, size, word in ((-1, 10, "n_users"), (2, 0, "size")):
        assert lib.srs_recforyou_ctr_host(None, None, None, p(q), n, size, *map(p, out)) == L.SRS_ERR_INVALID
        assert word in lib.srs_last_error().decode()
