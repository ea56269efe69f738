"""Recommended for you with every served CTR model (`RecForYou.set_user_features`, `srs_recforyou_ctr_host`,
DESIGN.md section 4.26): the 5 000 users of the golden ratings over the uf: / mf: hashes of the golden model samples,
every score bit for bit `CTRModel.rank_user`'s for that user and candidate, the order the oracle's fed those scores,
the float64 oracle (oracle/recforyou_features.py) within the feature-store tolerance; NeuralCF and two-tower models
through the new call; a 30 000-user, 70 000-movie page over several chunks; MODEL_RANGE; the rejections."""
import os

import numpy as np
import pytest

from oracle import recforyou as R
from oracle.recforyou_features import feature_score_fn, model_movie_id, read_history_keys
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import featurestore as FS
from sparrowrecsys_b200.features import GENRE_VOCAB
from sparrowrecsys_b200.model import CTRModel
from sparrowrecsys_b200.recforyou import RecForYou
from sparrowrecsys_b200.similar import SimilarMovies
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights
from test_gpu_recforyou import NCF_CASES, _check_rows, _oracle

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FEATURE_ATOL = 6e-5                     # test_featurestore.py: rank_user against the float64 forward

MODELS = {
    "embeddingmlp_tc": ("embeddingmlp", {}, {"embmlp_impl": "tc"}, "embmlp_tc"),
    "embeddingmlp_cudacore": ("embeddingmlp", {}, {"embmlp_impl": "cudacore"}, "embmlp_kernel"),
    "widendeep": ("widendeep", {}, None, None),
    "deepfm_e10": ("deepfm", {}, None, None),
    "deepfm_e16_tc": ("deepfm", {"emb_dim": 16}, {"deepfm_impl": "tc"}, "deepfm_tc"),
    "deepfm_e16_cudacore": ("deepfm", {"emb_dim": 16}, {"deepfm_impl": "cudacore"}, "deepfm_kernel"),
    "deepfm_v2": ("deepfm_v2", {}, None, None),
    "din_t5": ("din", {}, None, None),
    "din_wg_e32_t50": ("din", {"emb_dim": 32, "hist_len": 50}, None, "din_wg"),
    "dien": ("dien", {}, None, None),
}


def _golden_store():
    z = np.load(os.path.join(GOLDEN, "featureeng_model_samples.npz"))
    cols = {k: [str(x) for x in z[k].tolist()] for k in z.files if z[k].ndim == 1 and k != "text"}
    return FS.FeatureStore.from_samples(cols)


@pytest.fixture(scope="module")
def reference():
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    r = np.load(os.path.join(GOLDEN, "featureeng_ratings.npz"))
    movies = {"movieId": m["movieId"].astype(np.int32), "genres": [str(g) for g in m["genres"]]}
    ratings = {"userId": r["userId"].astype(np.int32), "movieId": r["movieId"].astype(np.int32),
               "rating": r["half"].astype(np.float64) / 2}
    users = np.unique(ratings["userId"])
    store = _golden_store()
    with_hash = np.array([bool(store.user_features(int(u))) for u in users])
    assert 0 < with_hash.sum() < len(users)               # both branches: users with and without a uf: hash
    cat = SimilarMovies(movies, ratings)
    page = RecForYou(cat, ratings)
    page.set_user_features(store)
    orc = _oracle(movies, ratings, None, None)
    cands = np.array([orc.cat.ids[c] for c in orc.candidates()], np.int32)
    yield users, cat, page, orc, store, cands, movies, ratings
    page.close()
    cat.close()


def _in_range(spec, store, uid, cands, n_table):
    """The page's MODEL_RANGE rule (oracle/recforyou_features.py)."""
    if not 0 <= uid < spec.n_users:
        return False
    if any(not 0 <= model_movie_id(spec, c) < spec.n_movies or not 0 <= c < n_table for c in cands.tolist()):
        return False
    typed = FS.parse_user_features(store.user_features(uid), max(spec.hist_len, 5))
    return all(0 <= model_movie_id(spec, typed[k]) < spec.n_movies for k in read_history_keys(spec))


def _rank_user_fn(model, store, cands, n_table):
    """score_fn of the oracle page from the device's own per-user path: rank_user's scores, widened to double."""
    def score(uid, movie_ids):
        assert np.array_equal(np.asarray(movie_ids, np.int32), cands)
        if not _in_range(model.spec, store, uid, cands, n_table):
            raise R.ModelRange(uid)
        return model.rank_user(uid, store.user_features(uid), cands, 800, return_scores=True)[2].astype(np.float64)
    return score


def _model(name, store):
    kind, kw, opts, kernel = MODELS[name]
    spec = default_spec(kind, **kw)
    W = init_weights(spec, 11)
    model = CTRModel(spec, W, options=opts)
    if kernel is not None:
        assert kernel in model.kernel_name, (name, model.kernel_name)
    table = FS.MovieFeatureTable.from_store(store, spec.n_movies)
    model.set_movie_table(table)
    return spec, W, model, table


@pytest.mark.parametrize("name", list(MODELS))
def test_every_reference_user(reference, name):
    users, _, page, orc, store, cands, _, _ = reference
    spec, W, model, table = _model(name, store)
    with model:
        fn = _rank_user_fn(model, store, cands, table.n_movies)
        out = page.recommend_arrays(users, 10, "nerualcf", model)
        assert (out[3] == R.OK).all() and (out[2] == 10).all()
        _check_rows(out, orc, users, 10, "nerualcf", fn)        # ids, statuses, counts; scores = rank_user's bits
        ref = feature_score_fn(spec, W, store, table, np.float64)
        rows = np.random.default_rng(3).choice(len(users), 40, replace=False)
        for q in rows:
            po = ref(int(users[q]), out[0][q])
            assert np.abs(out[1][q] - po).max() <= FEATURE_ATOL, (name, users[q])
        full = page.recommend_arrays(users[rows], 2000, "nerualcf", model)
        assert (full[2] == 800).all()
        _check_rows(full, orc, users[rows], 2000, "nerualcf", fn)


def _raw_ctr(page, cat, handle, q, size):
    lib = _lib.load()
    q = np.ascontiguousarray(q, np.int32)
    out = (np.zeros((len(q), size), np.int32), np.zeros((len(q), size), np.float64), np.zeros(len(q), np.int32),
           np.zeros(len(q), np.int32))
    p = lambda a: a.ctypes.data
    rc = lib.srs_recforyou_ctr_host(cat._h, page._h, handle, p(q), len(q), size, *map(p, out))
    return rc, out


@pytest.mark.parametrize("case", list(NCF_CASES))
def test_neuralcf_and_two_towers_through_the_ctr_call(reference, case):
    users, cat, page, _, _, _, _, _ = reference
    spec, W = NCF_CASES[case]()
    W = W if W is not None else init_weights(spec, 11)
    q = np.concatenate([users, [10 ** 6, -3]]).astype(np.int32)
    with CTRModel(spec, W) as model:
        want = page.recommend_arrays(q, 20, "nerualcf", model)
        rc, got = _raw_ctr(page, cat, model._h, q, 20)
        assert rc == _lib.SRS_OK
        assert all(a.tobytes() == b.tobytes() for a, b in zip(want, got))


def test_model_range(reference):
    users, cat, page, orc, store, cands, _, _ = reference
    # a small n_users
    spec = default_spec("deepfm", n_users=int(users[20]) + 1)
    with CTRModel(spec, init_weights(spec, 3)) as model:
        model.set_movie_table(FS.MovieFeatureTable.from_store(store, spec.n_movies))
        q = np.concatenate([users[:40], users[-40:], [10 ** 6]]).astype(np.int32)
        out = page.recommend_arrays(q, 10, "nerualcf", model)
        want = np.where(q <= users[20], R.OK, R.MODEL_RANGE)
        want[-1] = R.UNKNOWN_USER
        assert out[3].tolist() == want.tolist()
        bad = out[3] != R.OK
        assert not out[0][bad].any() and not out[1][bad].any() and not out[2][bad].any()
        _check_rows(out, orc, q, 10, "nerualcf", _rank_user_fn(model, store, cands, spec.n_movies))
    # a history id past n_movies: DIN reads userRatedMovie2, Wide&Deep only userRatedMovie1
    u = next(int(x) for x in users if store.user_features(int(x)).get("userRatedMovie2", "") not in ("", "0"))
    saved = store.user_features(u)
    store.backend.hset("uf:%d" % u, {"userRatedMovie2": "5000"})
    try:
        page.set_user_features(store)
        q = np.concatenate([[u], users[users != u][:2]]).astype(np.int32)
        for kind, first in (("din", R.MODEL_RANGE), ("dien", R.MODEL_RANGE), ("widendeep", R.OK)):
            spec = default_spec(kind)
            with CTRModel(spec, init_weights(spec, 4)) as model:
                model.set_movie_table(FS.MovieFeatureTable.from_store(store, spec.n_movies))
                out = page.recommend_arrays(q, 10, "nerualcf", model)
                assert out[3].tolist() == [first, R.OK, R.OK], kind
                _check_rows(out, orc, q, 10, "nerualcf", _rank_user_fn(model, store, cands, spec.n_movies))
    finally:
        store.backend.hset("uf:%d" % u, saved)
        page.set_user_features(store)
    # candidates past the movie table, and outside the model
    q = np.concatenate([users[:30], [10 ** 6]]).astype(np.int32)
    assert cands.max() >= 500
    for n_movies, rows in ((1001, 500), (500, 1001)):
        spec = default_spec("din", n_movies=n_movies)
        with CTRModel(spec, init_weights(spec, 5)) as model:
            model.set_movie_table(FS.MovieFeatureTable.from_store(store, rows))
            out = page.recommend_arrays(q, 10, "nerualcf", model)
            assert out[3].tolist() == [R.MODEL_RANGE] * 30 + [R.UNKNOWN_USER]
            assert not out[0].any() and not out[1].any() and not out[2].any()


def test_rejections_leave_both_handles_usable(reference):
    users, cat, page, _, store, _, movies, ratings = reference
    q = np.ascontiguousarray(users[:20], np.int32)
    spec, _, model, _ = _model("deepfm_e10", store)
    with model:
        before = page.recommend_arrays(q, 10, "nerualcf", model)
        lib = _lib.load()
        p = lambda a: a.ctypes.data
        ids, g, num, hist = (q[:2].copy(), np.zeros((2, 5), np.int32), np.zeros((2, 3), np.float32),
                             np.zeros((2, 5), np.int32))
        g[1, 3] = 19
        assert lib.srs_recforyou_users_set_features_host(page._h, 2, p(ids), p(g), p(num), p(hist)) == \
            _lib.SRS_ERR_RANGE
        with CTRModel(spec, init_weights(spec, 1)) as bare:                    # no movie table
            rc, out = _raw_ctr(page, cat, bare._h, q, 10)
            assert rc == _lib.SRS_ERR_INVALID and "srs_model_set_movie_features" in lib.srs_last_error().decode()
            assert not any(a.any() for a in out)
            with pytest.raises(ValueError, match="set_movie_table"):
                page.recommend(q, 10, "nerualcf", bare)
        with RecForYou(cat, ratings) as plain:                                 # no user features
            rc, _ = _raw_ctr(plain, cat, model._h, q, 10)
            assert rc == _lib.SRS_ERR_INVALID and "set_features" in lib.srs_last_error().decode()
            with pytest.raises(ValueError, match="set_user_features"):
                plain.recommend(q, 10, "nerualcf", model)
            assert (plain.recommend_arrays(q, 10, "default")[3] == R.OK).all()
        rc, _ = _raw_ctr(page, cat, model._h, q, 0)
        assert rc == _lib.SRS_ERR_INVALID
        after = page.recommend_arrays(q, 10, "nerualcf", model)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(before, after))
        assert model.rank_user(int(q[0]), store.user_features(int(q[0])), [1, 2], 2)[0].shape == (2,)


@pytest.fixture(scope="module")
def synthetic():
    rng = np.random.default_rng(23)
    n, n_users = 70_000, 30_000
    ids = rng.permutation(np.arange(1, 3 * n, dtype=np.int32))[:n]
    genres = [GENRE_VOCAB[g] for g in rng.integers(0, len(GENRE_VOCAB), n)]
    rm = ids[rng.integers(0, n, 400_000)]
    rs = rng.integers(1, 11, rm.shape[0]) / 2
    uids = rng.permutation(np.arange(1, n_users + 1, dtype=np.int32))
    ru = uids[rng.integers(0, n_users, rm.shape[0])]
    ru[:n_users] = uids
    movies = {"movieId": ids, "genres": genres}
    ratings = {"userId": ru, "movieId": rm.astype(np.int32), "rating": rs}
    store = FS.FeatureStore()
    for u in uids[rng.random(n_users) < 0.6].tolist():
        h = {"userRatedMovie%d" % k: str(int(ids[rng.integers(0, n)])) for k in range(1, 6)}
        h.update({"userGenre%d" % g: GENRE_VOCAB[int(rng.integers(0, len(GENRE_VOCAB)))] for g in range(1, 4)})
        h.update({"userRatingCount": str(int(rng.integers(1, 500))), "userAvgRating": "%.2f" % rng.uniform(1, 5),
                  "userRatingStddev": "%.2f" % rng.uniform(0, 2)})
        store.backend.hset("uf:%d" % u, h)
    n_movies = 3 * n
    table = FS.MovieFeatureTable(n_movies)
    for k in FS.MOVIE_STR_FIELDS:
        table.idx_cols[k][ids] = rng.integers(-1, len(GENRE_VOCAB), n)
    table.int_cols["movieRatingCount"][ids] = rng.integers(0, 10_000, n)
    table.int_cols["releaseYear"][ids] = rng.integers(1900, 2020, n)
    table.float_cols["movieAvgRating"][ids] = rng.uniform(0, 5, n).astype(np.float32)
    table.float_cols["movieRatingStddev"][ids] = rng.uniform(0, 2, n).astype(np.float32)
    cat = SimilarMovies(movies, ratings)
    page = RecForYou(cat, ratings)
    page.set_user_features(store)
    yield uids, page, store, table, n_movies
    page.close()
    cat.close()


@pytest.mark.parametrize("kind", ["din", "deepfm"])
def test_30000_users_over_several_chunks(synthetic, kind):
    uids, page, store, table, n_movies = synthetic
    spec = default_spec(kind, n_movies=n_movies, n_users=len(uids) + 1)
    with CTRModel(spec, init_weights(spec, 9)) as model:
        model.set_movie_table(table)
        q = np.concatenate([uids, [0, -1, len(uids) + 5]]).astype(np.int32)
        a = page.recommend_arrays(q, 20, "nerualcf", model)
        b = page.recommend_arrays(q, 20, "nerualcf", model)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
        assert (a[3][:len(uids)] == R.OK).all() and (a[3][len(uids):] == R.UNKNOWN_USER).all()
        # the candidates in page order: the default ranker lists them as they are
        cands = page.recommend_arrays(uids[:1], 800, "default")[0][0]
        rows = np.random.default_rng(4).choice(len(uids), 300, replace=False)
        for q_ in rows:
            uid = int(uids[q_])
            probs = model.rank_user(uid, store.user_features(uid), cands, 800, return_scores=True)[2]
            order = sorted(range(len(cands)), key=lambda i: (R.java_desc_key(float(probs[i])), int(cands[i])))[:20]
            assert a[0][q_].tolist() == cands[order].tolist(), uid
            assert a[1][q_].tobytes() == probs[order].astype(np.float64).tobytes(), uid
