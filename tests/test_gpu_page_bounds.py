"""The similar-movies and recommended-for-you pages on the device at their bounds (csrc/similar.cu, csrc/recforyou.cu,
DESIGN.md sections 4.23 - 4.26), on the catalogues of tests/test_page_bounds.py and the golden users:

* sim_query_kernel at sort widths 32 .. 8 192, 64 genres (bit 63), genres of 99 / 100 / 101 movies, MULTIPLE at
  np 2 048 and with every movie in both global lists, the genreless pair (NaN first);
* sim_emb_recall_kernel's two instantiations around their switch at a pool of 1 024, and a pool cut inside a tie;
* vectors of 1 .. 300 floats through every cosine (cosine.cuh), exact ties and pairs one ulp apart, checked bit
  for bit against the device's lane order (`warp_cosine_many`);
* RecForYou's sort at 1 .. 800 candidates with all three rankers, and the emb ranker's -1 rules;
* every "nerualcf" (EP, HP) instantiation through both host calls, the 48 KiB opt-in, the vocabulary edges;
* the CTR page's range rule (history positions at T = 3, 9, 10, ids past 2^24) and its chunks.
Every case checks statuses, counts, ids, the zero tail and scores bit for bit, and repeats a call.  The file runs
in about 31 s on an NVIDIA H100 80GB HBM3 at a 700 W power limit."""
import os
import re

import numpy as np
import pytest

from oracle import recforyou as R
from oracle import similar_movies as S
from oracle import similar_recall as SR
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import featurestore as FS
from sparrowrecsys_b200.features import GENRE_VOCAB, genre_to_index
from sparrowrecsys_b200.model import CTRModel
from sparrowrecsys_b200.ranking import rank_by_embedding
from sparrowrecsys_b200.recforyou import RecForYou
from sparrowrecsys_b200.similar import SimilarMovies
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights
from test_gpu_kernel_matrix import CSRC, MATRIX, TT, _case, _case_id, _seed
from test_gpu_recforyou import _check_rows, _device_score_fn, _oracle, _pairs
from test_gpu_recforyou_features import _golden_store, _raw_ctr, _rank_user_fn, reference  # noqa: F401 (fixture)
from test_gpu_similar import _check
from test_gpu_similar_recall import _check_multiple, _check_recall
from test_page_bounds import (WIDTHS, flat_catalogue, genre_catalogue, recall_oracle, small_multi_catalogue,
                              width_catalogue)

pytestmark = pytest.mark.gpu



def _ctr_batch_bytes():
    """recforyou.cu's kCtrBatchBytes, read from the source."""
    with open(os.path.join(CSRC, "recforyou.cu")) as f:
        m = re.search(r"constexpr size_t kCtrBatchBytes = \(size_t\)(\d+) << (\d+);", f.read())
    assert m, "kCtrBatchBytes not found in recforyou.cu"
    return int(m.group(1)) << int(m.group(2))


# The users of one chunk of the CTR page with DIN at T = 200: kCtrBatchBytes over one user's assembled rows.  The row
# size restates model.cu's packed_layout for DIN (movieId, userId, 200 history ids, 3 movie genres, 5 user genres,
# 7 numerics, 4 bytes each) over the 800 candidates; if that layout changes, this must follow it.
CTR_CHUNK_T200 = _ctr_batch_bytes() // (800 * 4 * (2 + 200 + 3 + 5 + 7))


def _same_bytes(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _rank_ratings(ratings, users):
    """`ratings` with a userId column, and one more line per user of `users` for a movie outside the catalogue:
    userMap holds every user of a line, and no average moves."""
    users = np.asarray(users, np.int32)
    return {"userId": np.concatenate([np.resize(users, len(ratings["movieId"])), users]),
            "movieId": np.concatenate([ratings["movieId"], np.full(len(users), 10 ** 8, np.int32)]),
            "rating": np.concatenate([ratings["rating"], np.full(len(users), 5.0)])}


# ---- sim_query_kernel ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind, np_", [(1, 32), (32, 32), (33, 64), (256, 256), (257, 512), (6400, 8192)])
def test_genre_candidates_at_each_sort_width(kind, np_):
    movies, ratings, emb, q, _ = genre_catalogue(kind)
    orc = recall_oracle(movies, ratings, emb)
    with SimilarMovies(movies, ratings, emb) as dev:
        for model in ("default", "emb"):
            for size in (1, np_ - 1, 10_000):
                _, _, count, status = _check(dev, orc, q, size, model)
                assert status[-1] == S.UNKNOWN_MOVIE
            assert _same_bytes(dev.recommend_arrays(q, np_, model), dev.recommend_arrays(q, np_, model))
        if kind == 6400:               # the all-genre movie: 64 lists of 100, itself in each; {G40, G63}: 2 x 100 - 1
            assert count[0] == 64 * 99 and count[3] == 199
            for size in (1, 2047, 10_000):                     # MULTIPLE: 64 x 20 + 2 x 100 = 1 480, np 2 048
                for model in ("default", "emb"):
                    _check_multiple(dev, orc, q, size, model)


def test_multiple_candidates_of_a_small_catalogue_and_the_genreless_pair():
    movies, ratings, emb = small_multi_catalogue()
    orc = recall_oracle(movies, ratings, emb)
    q = np.concatenate([movies["movieId"], [10 ** 6]]).astype(np.int32)
    with SimilarMovies(movies, ratings, emb) as dev:
        for model in ("default", "emb"):
            for size in (1, 39, 100):
                _, scores, count, status = _check_multiple(dev, orc, q, size, model)
                assert (status[:-1] == S.OK).all() and (count[:-1] == min(size, 39)).all()
            assert _same_bytes(dev.recommend_arrays(q, 50, model, "multiple"),
                               dev.recommend_arrays(q, 50, model, "multiple"))
        ids, scores, _, _ = dev.recommend_arrays(q[:1], 39, "default", "multiple")
        nan = np.isnan(scores[0])
        assert nan.sum() == 9 and nan[:9].all() and ids[0, :9].tolist() == sorted(ids[0, :9].tolist())


# ---- sim_emb_recall_kernel -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 31, 32, 1023, 1024, 1025, 10_001])
def test_embedding_recall_pools(n):
    movies, ratings, emb = flat_catalogue(n)
    ids, vec = emb
    zero = min(2, n - 1)
    if n > 1:
        vec[zero] = 0.0                # a zero-vector query: every score NaN, last
    orc = recall_oracle(movies, ratings, emb)
    pool = len(orc.get_movies(SR.POOL, "rating"))
    assert pool == min(n, SR.POOL)
    q = np.array([ids[0], ids[zero], ids[-1], ids[n // 2], 10 ** 6, ids[0]], np.int32)
    cache = {}
    with SimilarMovies(movies, ratings, emb) as dev:
        for size in (1, pool, pool + 1):
            _, scores, count, status = _check_recall(dev, orc, q, size, cache)
            assert (count[:4] == min(size, pool)).all() and status[4] == S.UNKNOWN_MOVIE
        if n > 1:
            assert np.isnan(scores[1, :pool]).all()
        assert _same_bytes(dev.retrieve_by_embedding_arrays(q, pool), dev.retrieve_by_embedding_arrays(q, pool))
    if n > SR.POOL:                    # only the movie cut from the pool has a vector: its pool is all -1, by id
        cut = orc.get_movies(SR.POOL + 1, "rating")[-1]
        lone = (ids[cut:cut + 1], vec[cut:cut + 1])
        orc1 = recall_oracle(movies, ratings, lone)
        with SimilarMovies(movies, ratings, lone) as dev:
            out = _check_recall(dev, orc1, ids[cut:cut + 1], SR.POOL, {})
            assert (out[1][0] == -1.0).all() and (np.diff(out[0][0]) > 0).all()


# ---- vector widths -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", WIDTHS)
def test_vector_widths_through_every_cosine(dim):
    movies, ratings, emb = width_catalogue(dim)
    ids, vec = emb
    rows = [0, 10, 20, 5, 15, 25, 30, 31] + list(range(40, 300, 23))
    q = ids[rows]
    users = np.arange(1, 41, dtype=np.int32)
    uvec = vec[(np.arange(40) * 7) % 300].copy()
    uvec[0], uvec[1] = vec[0], vec[31]     # a duplicated movie vector (exact ties); past 33 the ulp pair's ones
    uemb = (users, uvec)
    rat = _rank_ratings(ratings, users)
    orc = recall_oracle(movies, ratings, emb)
    rorc = _oracle(movies, rat, emb, uemb)
    with SimilarMovies(movies, ratings, emb) as dev, RecForYou(dev, rat, uemb) as page:
        _check(dev, orc, q, 300, "emb")
        _check_multiple(dev, orc, q, 300, "emb")
        _check_recall(dev, orc, q, 300, {})
        out = page.recommend_arrays(users, 300, "emb")
        _check_rows(out, rorc, users, 300, "emb")
        assert _same_bytes(out, page.recommend_arrays(users, 300, "emb"))
        if dim >= 34:                  # the device's lane order, not the Java's
            r = list(q).index(ids[31])
            got = dict(zip(*[a[r] for a in dev.recommend_arrays(q, 300, "emb")[:2]]))
            assert got[ids[30]] == S.warp_cosine_many(vec[31], vec[30:31])[0] != S.java_cosine_many(vec[31],
                                                                                                   vec[30:31])[0]
    # ranking.rank_by_embedding: util.cu's cosine_kernel (float32 of the same double) and the top-k
    for r in (0, 31, 77):
        idx, top = rank_by_embedding(vec[r], vec, 40)
        want = S.warp_cosine_many(vec[r], vec).astype(np.float32)
        order = sorted(range(len(vec)), key=lambda i: (R.java_desc_key(float(want[i])), i))[:40]
        assert idx.tolist() == order and top.tobytes() == want[order].tobytes(), (dim, r)


# ---- RecForYou -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 31, 32, 33, 512, 513, 800])
def test_recforyou_sort_at_each_width(n):
    movies, ratings, emb = flat_catalogue(n)
    users = np.arange(1, 41, dtype=np.int32)
    rng = np.random.default_rng(n)
    uvec = rng.standard_normal((40, 16)).astype(np.float32)
    uvec[3] = 0.0                                              # NaN for every candidate
    uemb = (users[:30], uvec[:30])                             # users 31..40: no vector, all -1
    rat = _rank_ratings(ratings, users)
    orc = _oracle(movies, rat, emb, uemb)
    q = np.concatenate([users, [0, 10 ** 6], users[:3]]).astype(np.int32)
    spec = default_spec("neuralcf", n_movies=int(movies["movieId"].max()) + 1, n_users=41)
    with SimilarMovies(movies, ratings, emb) as cat, RecForYou(cat, rat, uemb) as page, \
            CTRModel(spec, init_weights(spec, n)) as model:
        for name in ("default", "emb", "nerualcf"):
            for size in (1, n, n + 1):
                out = page.recommend_arrays(q, size, name, model)
                _check_rows(out, orc, q, size, name, _device_score_fn(model) if name == "nerualcf" else None)
                assert (out[3][40:42] == R.UNKNOWN_USER).all() and (out[2][:40] == min(size, n)).all()
            assert _same_bytes(out, page.recommend_arrays(q, n + 1, name, model))


def test_emb_rules():
    movies, ratings, emb = flat_catalogue(200)
    users = np.arange(1, 21, dtype=np.int32)
    rat = _rank_ratings(ratings, users)
    rng = np.random.default_rng(1)
    cases = {
        "other dim": (emb, (users, rng.standard_normal((20, 8)).astype(np.float32))),
        "no movie vectors": (None, (users, rng.standard_normal((20, 16)).astype(np.float32))),
        "unknown user's line": (emb, (np.array([10 ** 6, 5], np.int32),
                                      rng.standard_normal((2, 16)).astype(np.float32))),
    }
    q = np.concatenate([users, [10 ** 6]]).astype(np.int32)
    for what, (memb, uemb) in cases.items():
        orc = _oracle(movies, rat, memb, uemb)
        with SimilarMovies(movies, ratings, memb) as cat, RecForYou(cat, rat, uemb) as page:
            out = page.recommend_arrays(q, 300, "emb")
            _check_rows(out, orc, q, 300, "emb")
            minus = [u for u in range(20) if what != "unknown user's line" or users[u] != 5]
            assert (out[1][minus, :200] == -1.0).all() and (np.diff(out[0][minus, :200], axis=1) > 0).all(), what
            assert out[3][-1] == R.UNKNOWN_USER


# ---- "nerualcf": every instantiation ------------------------------------------------------------------------------
NCF_PAGE_CASES = [c for c in MATRIX if c.model in ("neuralcf", "twotowers")] + [
    _case("twotowers", TT, emb_dim=12, hidden=(16,), final_dense=False),
    _case("twotowers", TT, emb_dim=1, hidden=(32, 17), final_dense=True),
    # 16 KiB of sort and an 8 392-float blob: rfy_ncf_kernel's shared memory past 48 KiB
    *[_case("twotowers", TT, emb_dim=64, hidden=(32, 32, 32), final_dense=fd) for fd in (True, False)]]


@pytest.mark.parametrize("case", NCF_PAGE_CASES, ids=_case_id)
def test_nerualcf_instantiation(reference, case):
    users, cat, page, orc, _, cands, _, _ = reference
    spec = default_spec(case.model, n_movies=int(cands.max()) + 1, n_users=int(users.max()) + 1, **case.over)
    q = np.concatenate([users[::16], [10 ** 6]]).astype(np.int32)            # 313 users: several blocks
    with CTRModel(spec, init_weights(spec, _seed(case))) as model:
        out = page.recommend_arrays(q, 10, "nerualcf", model)
        rc, got = _raw_ctr(page, cat, model._h, q, 10)
        assert rc == _lib.SRS_OK and _same_bytes(out, got)
        assert (out[3][:-1] == R.OK).all() and out[3][-1] == R.UNKNOWN_USER
        u, m = _pairs(q[:-1], tuple(a[:-1] for a in out))
        p = model.predict({"userId": u, "movieId": m})[:, 0]
        got_scores = np.concatenate([out[1][r, :10] for r in range(len(q) - 1)])
        assert got_scores.tobytes() == p.astype(np.float64).tobytes()
        full = page.recommend_arrays(q[:12], 2000, "nerualcf", model)
        _check_rows(full, orc, q[:12], 2000, "nerualcf", _device_score_fn(model))
        assert _same_bytes(out, page.recommend_arrays(q, 10, "nerualcf", model))


@pytest.mark.parametrize("kind", ["neuralcf", "twotowers"])
def test_nerualcf_vocabulary_edges(reference, kind):
    users, cat, page, _, _, cands, _, _ = reference
    top_m, top_u = int(cands.max()), int(users.max())
    q = np.concatenate([users[:5], users[-5:]]).astype(np.int32)
    for n_movies, n_users, want in ((top_m + 1, top_u + 1, [R.OK] * 10),
                                    (top_m, top_u + 1, [R.MODEL_RANGE] * 10),
                                    (top_m + 1, top_u, [R.OK] * 9 + [R.MODEL_RANGE])):
        spec = default_spec(kind, n_movies=n_movies, n_users=n_users)
        with CTRModel(spec, init_weights(spec, 2)) as model:
            out = page.recommend_arrays(q, 10, "nerualcf", model)
            assert out[3].tolist() == want, (n_movies, n_users)
            bad = out[3] != R.OK
            assert not out[0][bad].any() and not out[1][bad].any() and not out[2][bad].any()
            assert _same_bytes(out, _raw_ctr(page, cat, model._h, q, 10)[1])


# ---- the CTR page: the range rule --------------------------------------------------------------------------------
def _full_history_users(store, users, k):
    full = lambda f: all(f.get("userRatedMovie%d" % j, "") not in ("", "0") for j in range(1, 6))
    return [int(u) for u in users if full(store.user_features(int(u)))][:k]


def _ctr_page(cat, ratings, edits):
    """A page over a fresh golden store with `edits` ({user: {key: value}}) applied."""
    store = _golden_store()
    for u, h in edits.items():
        store.backend.hset("uf:%d" % u, h)
    page = RecForYou(cat, ratings)
    page.set_user_features(store)
    return page, store


def _check_ctr(page, orc, model, store, cands, q, table_rows, want):
    out = page.recommend_arrays(q, 10, "nerualcf", model)
    assert out[3].tolist() == want
    _check_rows(out, orc, q, 10, "nerualcf", _rank_user_fn(model, store, cands, table_rows))
    assert _same_bytes(out, page.recommend_arrays(q, 10, "nerualcf", model))
    return out


@pytest.mark.parametrize("kind", ["din", "dien"])
def test_ctr_range_rule_follows_the_history_positions(reference, kind):
    users, cat, _, orc, store0, cands, _, ratings = reference
    a, b, c = _full_history_users(store0, users, 3)
    q = np.array([a, b, c], np.int32)
    for T, key, first in ((3, "userRatedMovie4", R.OK), (3, "userRatedMovie5", R.OK),
                          (9, "userRatedMovie2", R.MODEL_RANGE), (9, "userRatedMovie5", R.MODEL_RANGE),
                          (10, "userRatedMovie2", R.MODEL_RANGE), (10, "userRatedMovie5", R.MODEL_RANGE)):
        page, store = _ctr_page(cat, ratings, {a: {key: "5000"}})
        spec = default_spec(kind, hist_len=T)
        with page, CTRModel(spec, init_weights(spec, T)) as model:
            table = FS.MovieFeatureTable.from_store(store, spec.n_movies)
            model.set_movie_table(table)
            _check_ctr(page, orc, model, store, cands, q, table.n_movies, [first, R.OK, R.OK])


def test_ctr_range_rule_past_2_24(reference):
    from test_gpu_seq_axis import _big_table
    from test_seq_axis import BIG_VOCAB, ROUNDS_DOWN, ROUNDS_OUT
    users, cat, _, orc, store0, cands, _, ratings = reference
    a, b, c = _full_history_users(store0, users, 3)
    q = np.array([a, b, c], np.int32)
    page, store = _ctr_page(cat, ratings, {a: {"userRatedMovie3": str(ROUNDS_OUT)},
                                           b: {"userRatedMovie3": str(ROUNDS_DOWN)}})
    with page:
        spec = default_spec("din", emb_dim=12, n_movies=BIG_VOCAB)
        W = init_weights(spec, 24, skip=("embedding",))
        W["embedding"] = _big_table(12)                        # 2^24 + 4 rows on the device, lent to the model
        with CTRModel(spec, W) as model:
            model.set_movie_table(FS.MovieFeatureTable.from_store(store, 1001))
            _check_ctr(page, orc, model, store, cands, q, 1001, [R.MODEL_RANGE, R.OK, R.OK])
        del W
        spec = default_spec("widendeep")                       # reads userRatedMovie1 only
        with CTRModel(spec, init_weights(spec, 25)) as model:
            model.set_movie_table(FS.MovieFeatureTable.from_store(store, spec.n_movies))
            _check_ctr(page, orc, model, store, cands, q, spec.n_movies, [R.OK, R.OK, R.OK])


# ---- the CTR page: chunks ------------------------------------------------------------------------------------------
def test_ctr_chunks_with_failing_users_at_every_edge(reference):
    users, cat, _, orc, store0, cands, _, ratings = reference
    rng = np.random.default_rng(200)
    poisoned = [int(u) for u in rng.choice(users, 300, replace=False)]
    page, store = _ctr_page(cat, ratings, {u: {"userRatedMovie1": "5000"} for u in poisoned})
    spec = default_spec("din", hist_len=200)
    C = CTR_CHUNK_T200
    with page, CTRModel(spec, init_weights(spec, 200)) as model:
        table = FS.MovieFeatureTable.from_store(store, spec.n_movies)
        model.set_movie_table(table)
        bad = set(poisoned)
        passing = [int(u) for u in users if int(u) not in bad] + [int(u) for u in rng.choice(users, 300)
                                                                   if int(u) not in bad]
        failing = poisoned + [10 ** 6 + k for k in range(100)] + [-k for k in range(1, 50)]
        q, f, edge_rows = [], 0, []
        for j, u in enumerate(passing):         # a failing query before the first and the last user of each chunk
            if j % C in (0, C - 1) or rng.random() < 0.05:
                q.append(failing[f % len(failing)])
                f += 1
            if j % C in (0, C - 1):
                edge_rows.append(len(q))
            q.append(u)
        q = np.array(q, np.int32)
        assert len(passing) > 12 * C
        out = page.recommend_arrays(q, 10, "nerualcf", model)
        want = np.where(np.isin(q, passing), R.OK, np.where(np.isin(q, poisoned), R.MODEL_RANGE, R.UNKNOWN_USER))
        assert out[3].tolist() == want.tolist()
        bad_rows = out[3] != R.OK
        assert not out[0][bad_rows].any() and not out[1][bad_rows].any() and not out[2][bad_rows].any()
        fn = _rank_user_fn(model, store, cands, table.n_movies)
        sample = sorted(set(edge_rows) | set(rng.choice(len(q), 60, replace=False).tolist()))
        _check_rows(out, orc, q, 10, "nerualcf", fn, rows=sample)
        full = page.recommend_arrays(q[sample[:8]], 800, "nerualcf", model)
        _check_rows(full, orc, q[sample[:8]], 800, "nerualcf", fn)
        # pass counts 386 k - 1, 386 k, 386 k + 1: the same rows as the whole call's
        ok_rows = np.flatnonzero(~bad_rows)
        for k in (1, 2):
            for n_pass in (C * k - 1, C * k, C * k + 1):
                end = ok_rows[n_pass - 1] + 1
                part = page.recommend_arrays(q[:end], 10, "nerualcf", model)
                assert _same_bytes(part, tuple(a[:end] for a in out)), n_pass
        # nobody passes; exactly one passes
        rc, none = _raw_ctr(page, cat, model._h, np.array(failing[:50], np.int32), 10)
        assert rc == _lib.SRS_OK and not none[0].any() and not none[1].any() and not none[2].any()
        assert (none[3] != R.OK).all()
        one = np.array([failing[0], passing[7], failing[1]], np.int32)
        rc, got = _raw_ctr(page, cat, model._h, one, 10)
        assert rc == _lib.SRS_OK and got[3].tolist() == [R.MODEL_RANGE, R.OK, R.MODEL_RANGE]
        r7 = list(q).index(passing[7])
        assert got[0][1].tobytes() == out[0][r7].tobytes() and got[1][1].tobytes() == out[1][r7].tobytes()


# ---- the CTR page: the users' uf: rows ----------------------------------------------------------------------------
def _feature_rows(store, rows):
    """srs_recforyou_users_set_features_host's arrays for `rows` [(user id, fields)], typed as set_user_features
    types a hash."""
    ids, genres, nums, hist = [], [], [], []
    for u, fields in rows:
        t = FS.parse_user_features(fields)
        ids.append(u)
        genres.append([int(genre_to_index([t["userGenre%d" % (g + 1)]])[0]) for g in range(5)])
        nums.append([t["userAvgRating"], np.float32(t["userRatingCount"]), t["userRatingStddev"]])
        hist.append([t["userRatedMovie%d" % (k + 1)] for k in range(5)])
    return [np.ascontiguousarray(np.array(x, dt)) for x, dt in
            ((ids, np.int32), (genres, np.int32), (nums, np.float32), (hist, np.int32))]


def test_user_feature_rows(reference):
    users, cat, _, orc, store0, cands, _, ratings = reference
    a, b, c, d = _full_history_users(store0, users, 4)
    fa, fb, fc = store0.user_features(a), dict(store0.user_features(b)), dict(store0.user_features(c))
    fb["userGenre1"] = GENRE_VOCAB[18]                         # the last index of the vocabulary: accepted
    rows = _feature_rows(store0, [(a, store0.user_features(d)), (10 ** 6, fa), (b, fb), (c, fc), (a, fa)])
    rows[1][3, 1] = -7                                         # c's userGenre2: read as missing
    del fc["userGenre2"]
    want = FS.FeatureStore()                                   # what the page must have read, user by user
    for u, f in ((a, fa), (b, fb), (c, fc)):
        want.backend.hset("uf:%d" % u, f)
    spec = default_spec("deepfm")
    with RecForYou(cat, ratings) as page, CTRModel(spec, init_weights(spec, 6)) as model:
        _lib.check(_lib.load().srs_recforyou_users_set_features_host(page._h, len(rows[0]),
                                                                     *[x.ctypes.data for x in rows]))
        page.has_user_features = True
        table = FS.MovieFeatureTable.from_store(store0, spec.n_movies)
        model.set_movie_table(table)
        q = np.array([a, b, c, d], np.int32)                   # d has no row: an empty hash's values
        _check_ctr(page, orc, model, want, cands, q, table.n_movies, [R.OK] * 4)
