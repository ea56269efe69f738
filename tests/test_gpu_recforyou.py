"""Recommended for you on the device (`RecForYou`, `srs_recforyou_host`, csrc/recforyou.cu) against the oracle
(oracle/recforyou.py): the 5 000 users of the golden ratings with the emb and default rankers, the "nerualcf" ranker
with the shipped NeuralCF and two-tower models and deeper synthetic ones (every score bit for bit the model's
`predict` of that pair), users and candidates outside the model, a synthetic catalogue past 65 536 movies with 30 000
users, the rejections and repeat calls.  Cosines are checked bit for bit against the oracle summing in the device's
lane order (`warp_cosine_many`)."""
import os

import numpy as np
import pytest

from conftest import load_golden_weights
from oracle import recforyou as R
from oracle import similar_movies as S
from oracle.similar_recall import RecallCatalogue
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200.model import CTRModel
from sparrowrecsys_b200.ranking import load_embeddings_csv
from sparrowrecsys_b200.recforyou import RecForYou
from sparrowrecsys_b200.similar import SimilarMovies, genre_lists
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights
from test_gpu_similar import score_bits

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PROB_ATOL = 2e-5                        # test_gpu_parity.py: the CUDA path against the float64 forward


def _oracle(movies, ratings, emb, uemb):
    cat = RecallCatalogue(movies["movieId"], genre_lists(list(movies["genres"])), ratings["movieId"],
                          np.asarray(ratings["rating"], np.float32), *(emb if emb is not None else (None, None)),
                          cosine=S.warp_cosine_many)
    return R.RecForYou(cat, ratings["userId"], *(uemb if uemb is not None else (None, None)),
                       cosine=S.warp_cosine_many)


def _check_rows(out, orc, users, size, model, score_fn=None, rows=None):
    """Rows `rows` (all by default) of the device's `out` against the oracle's lists."""
    ids, scores, count, status = out
    for q in (range(len(users)) if rows is None else rows):
        uid = int(users[q])
        oi, osc, ost = orc.rec_list(uid, size, model, score_fn)
        assert status[q] == ost, (uid, status[q], ost)
        assert count[q] == len(oi), (uid, count[q], len(oi))
        assert ids[q, :count[q]].tolist() == oi, (uid, model, size)
        assert not ids[q, count[q]:].any() and not scores[q, count[q]:].any()
        if model != "nerualcf" or score_fn is not None:
            assert scores[q, :count[q]].tobytes() == score_bits(osc), (uid, model, size)


@pytest.fixture(scope="module")
def reference():
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    r = np.load(os.path.join(GOLDEN, "featureeng_ratings.npz"))
    movies = {"movieId": m["movieId"].astype(np.int32), "genres": [str(g) for g in m["genres"]]}
    ratings = {"userId": r["userId"].astype(np.int32), "movieId": r["movieId"].astype(np.int32),
               "rating": r["half"].astype(np.float64) / 2}
    emb = load_embeddings_csv(os.path.join(GOLDEN, "item2vecEmb.csv"))
    z = np.load(os.path.join(GOLDEN, "item2vec_user_emb.npz"))
    uemb = (z["user"].astype(np.int32),
            np.array([[float(v) for v in ln.split(":")[1].split()] for ln in z["line"].tolist()], np.float32))
    users = np.unique(ratings["userId"])
    assert len(users) == 5000 and len(movies["movieId"]) == 982
    cat = SimilarMovies(movies, ratings, emb)
    page = RecForYou(cat, ratings, uemb)
    yield users, cat, page, _oracle(movies, ratings, emb, uemb)
    page.close()
    cat.close()


@pytest.mark.parametrize("model", ["default", "emb"])
@pytest.mark.parametrize("size", [10, 2000])
def test_every_reference_user(reference, model, size):
    users, _, page, orc = reference
    out = page.recommend_arrays(users, size, model)
    assert (out[3] == R.OK).all() and (out[2] == min(size, 800)).all()
    _check_rows(out, orc, users, size, model)


def _pairs(users, out):
    ids, _, count, _ = out
    u = np.repeat(np.asarray(users, np.int32), count)
    m = np.concatenate([ids[q, :count[q]] for q in range(len(users))])
    return u, m


def _device_score_fn(model):
    return lambda u, movies: model.predict({"userId": np.full(len(movies), u, np.int32),
                                            "movieId": np.asarray(movies, np.int32)})[:, 0].astype(np.float64)


NCF_CASES = {
    "neuralcf_002": lambda: (default_spec("neuralcf"), load_golden_weights("neuralcf_002")),
    "mlprec_005": lambda: (default_spec("twotowers", hidden=(10,), final_dense=False), load_golden_weights("mlprec_005")),
    "neuralcf_deep": lambda: (default_spec("neuralcf", emb_dim=64, hidden=(32, 24, 32), n_movies=1001, n_users=6000),
                              None),
    "twotowers_dense": lambda: (default_spec("twotowers", hidden=(16, 8), final_dense=True, n_movies=1001,
                                             n_users=6000), None),
}


@pytest.mark.parametrize("case", list(NCF_CASES))
def test_nerualcf_scores_are_the_models_bits(reference, case):
    users, _, page, orc = reference
    spec, W = NCF_CASES[case]()
    W = W if W is not None else init_weights(spec, 11)
    with CTRModel(spec, W) as model:
        out = page.recommend_arrays(users, 10, "nerualcf", model)
        assert (out[3] == R.OK).all() and (out[2] == 10).all()
        u, m = _pairs(users, out)
        p = model.predict({"userId": u, "movieId": m})[:, 0]
        got = np.concatenate([out[1][q, :10] for q in range(len(users))])
        assert got.tobytes() == p.astype(np.float64).tobytes()
        ref = R.ctr_score_fn(spec, W, np.float64)
        po = np.concatenate([ref(int(x), out[0][q, :10]) for q, x in enumerate(users)])
        assert np.abs(got - po).max() <= PROB_ATOL
        # whole lists for a sample: the order is the oracle's fed the device's own scores
        rows = np.random.default_rng(5).choice(len(users), 60, replace=False)
        full = page.recommend_arrays(users[rows], 2000, "nerualcf", model)
        assert (full[2] == 800).all()
        _check_rows(full, orc, users[rows], 2000, "nerualcf", _device_score_fn(model))


def test_users_and_candidates_outside_the_model(reference):
    users, _, page, orc = reference
    q = np.concatenate([users[:40], users[-40:], [10 ** 6, -3]]).astype(np.int32)
    spec = default_spec("neuralcf", n_movies=1001, n_users=int(users[20]) + 1)
    W = init_weights(spec, 3)
    with CTRModel(spec, W) as model:
        out = page.recommend_arrays(q, 10, "nerualcf", model)
        want = np.where(q <= users[20], R.OK, R.MODEL_RANGE)
        want[-2:] = R.UNKNOWN_USER
        assert out[3].tolist() == want.tolist()
        bad = out[3] != R.OK
        assert not out[0][bad].any() and not out[1][bad].any() and not out[2][bad].any()
        _check_rows(out, orc, q, 10, "nerualcf", R.ctr_score_fn(spec, W), rows=np.flatnonzero(bad))
    spec = default_spec("neuralcf", n_movies=500, n_users=30001)     # candidates reach movie id 1000
    with CTRModel(spec, init_weights(spec, 4)) as model:
        out = page.recommend_arrays(q, 10, "nerualcf", model)
        assert out[3].tolist() == [R.MODEL_RANGE] * (len(q) - 2) + [R.UNKNOWN_USER] * 2
        assert not out[0].any() and not out[2].any()
    assert (page.recommend_arrays(q[:5], 10, "default")[3] == R.OK).all()


def test_a_second_call_gives_the_same_bits(reference):
    users, _, page, _ = reference
    spec, W = NCF_CASES["neuralcf_002"]()
    with CTRModel(spec, W) as model:
        for model_name in ("default", "emb", "nerualcf"):
            a = page.recommend_arrays(users, 50, model_name, model)
            b = page.recommend_arrays(users, 50, model_name, model)
            assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_rejections_leave_both_handles_usable(reference):
    users, cat, page, _ = reference
    q = np.ascontiguousarray(users[:20], np.int32)
    before = page.recommend_arrays(q, 10, "emb")
    lib = _lib.load()
    out = [np.zeros(200, np.int32), np.zeros(200, np.float64), np.zeros(20, np.int32), np.zeros(20, np.int32)]
    p = lambda a: a.ctypes.data
    spec = default_spec("deepfm")
    with CTRModel(spec, init_weights(spec, 1)) as deepfm:
        for model, ranker, size, arrays in ((None, _lib.SRS_RECFORYOU_EMB, 0, out),
                                            (None, _lib.SRS_RECFORYOU_DEFAULT, -1, out),
                                            (None, 7, 10, out),
                                            (None, _lib.SRS_RECFORYOU_NEURALCF, 10, out),
                                            (deepfm._h, _lib.SRS_RECFORYOU_NEURALCF, 10, out),
                                            (None, _lib.SRS_RECFORYOU_EMB, 10, [None] + out[1:]),
                                            (None, _lib.SRS_RECFORYOU_EMB, 10, out[:3] + [None])):
            arr = [None if a is None else p(a) for a in arrays]
            assert lib.srs_recforyou_host(cat._h, page._h, model, ranker, p(q), 20, size, *arr) == \
                _lib.SRS_ERR_INVALID
        assert lib.srs_recforyou_host(cat._h, page._h, None, 0, None, 20, 10, *map(p, out)) == _lib.SRS_ERR_INVALID
        assert lib.srs_recforyou_host(None, page._h, None, 0, p(q), 20, 10, *map(p, out)) == _lib.SRS_ERR_INVALID
        assert lib.srs_recforyou_host(cat._h, None, None, 0, p(q), 20, 10, *map(p, out)) == _lib.SRS_ERR_INVALID
        with pytest.raises(ValueError):
            page.recommend(q, 10, "nerualcf")
        with pytest.raises(ValueError):
            page.recommend(q, 10, "nerualcf", deepfm)
        with pytest.raises(ValueError):
            page.recommend(q, 0, "emb")
    import torch
    if torch.cuda.device_count() > 1:
        spec = default_spec("neuralcf")
        with CTRModel(spec, init_weights(spec, 1), device=1) as other:
            with pytest.raises(_lib.SrsInvalidError, match="device"):
                page.recommend(q, 10, "nerualcf", other)
    after = page.recommend_arrays(q, 10, "emb")
    assert all(x.tobytes() == y.tobytes() for x, y in zip(before, after))


def test_a_treeified_catalogue_is_rejected():
    ids = np.array(list(range(1, 61)) + [1024 * k for k in range(1, 10)], np.int32)
    movies = {"movieId": ids, "genres": ["A"] * len(ids)}
    ratings = {"userId": np.array([1, 2], np.int32), "movieId": ids[:2], "rating": np.array([4.0, 3.0])}
    with SimilarMovies(movies, ratings) as cat, RecForYou(cat, ratings) as page:
        for model in ("default", "emb"):
            with pytest.raises(_lib.SrsInvalidError, match="treeified"):
                page.recommend([1, 2], 5, model)
    ids = ids[:60]
    movies = {"movieId": ids, "genres": ["A"] * len(ids)}
    with SimilarMovies(movies, ratings) as cat, RecForYou(cat, ratings) as page:
        r = page.recommend([1, 2, 3], 5, "default")
        assert [x.status for x in r] == [R.OK, R.OK, R.UNKNOWN_USER]
        assert r[0].movie_ids.tolist() == [1, 2, 3, 4, 5] and r[0].scores.tolist() == [60.0, 59.0, 58.0, 57.0, 56.0]


@pytest.fixture(scope="module")
def synthetic():
    rng = np.random.default_rng(17)
    n, n_users, dim = 70_000, 30_000, 16
    ids = rng.permutation(np.arange(1, 3 * n, dtype=np.int32))[:n]
    genres = ["G%d" % g for g in rng.integers(0, 20, n)]
    # 1 000 movies average exactly 5.0: the 800 candidates are all tied, chosen and ordered by movieMap's order
    top = rng.choice(n, 1000, replace=False)
    rm = ids[np.repeat(top, 2)].tolist()
    rs = [5.0] * len(rm)
    other = rng.integers(0, n, 600_000)
    other = other[~np.isin(other, top)]
    rm += ids[other].tolist()
    rs += (rng.integers(1, 10, other.shape[0]) / 2).tolist()
    user_ids = rng.permutation(np.unique(rng.integers(8, 2 ** 31 - 1, n_users * 2).astype(np.int32)))[:n_users]
    ru = user_ids[rng.integers(0, n_users, len(rm))]
    ru[:n_users] = user_ids                                         # every user rates once at least
    ru = rng.permutation(ru)
    movies = {"movieId": ids, "genres": genres}
    ratings = {"userId": ru, "movieId": np.array(rm, np.int32), "rating": np.array(rs)}
    has = rng.random(n) < 0.7
    emb = (ids[has], rng.standard_normal((int(has.sum()), dim)).astype(np.float32))
    known = np.unique(ru)
    with_vec = rng.choice(known, len(known) // 2, replace=False)
    vec = rng.standard_normal((len(with_vec), dim)).astype(np.float32)
    vec[200:250] = 0.0                                              # zero vectors: NaN for every candidate with one
    extra = np.array([5, 7], np.int32)                              # lines of users without ratings
    uemb = (np.concatenate([with_vec, extra, with_vec[:100]]).astype(np.int32),
            np.concatenate([vec, np.ones((2, dim), np.float32), vec[100:200]]))   # later lines win
    cat = SimilarMovies(movies, ratings, emb)
    page = RecForYou(cat, ratings, uemb)
    yield known, with_vec, cat, page, _oracle(movies, ratings, emb, uemb)
    page.close()
    cat.close()


def test_synthetic_catalogue_and_30000_users(synthetic):
    known, with_vec, _, page, orc = synthetic
    assert len(known) == 30_000 and len(orc.cat.ids) > 65_536
    cands = orc.candidates()
    assert {orc.cat.avg[c] for c in cands} == {5.0} and sorted(cands) != cands     # tied: HashMap order, not load
    rng = np.random.default_rng(2)
    q = np.concatenate([known, with_vec[:60], [5, 7, 0, -1, 2 ** 31 - 1], known[:10]]).astype(np.int32)
    special = np.concatenate([np.arange(len(known), len(q)), rng.choice(len(known), 400, replace=False)])
    for model in ("default", "emb"):
        for size in (20, 1000):
            out = page.recommend_arrays(q, size, model)
            assert (out[3][:len(known)] == R.OK).all() and (out[3][len(known) + 60:-10] == R.UNKNOWN_USER).all()
            if model == "default":
                _check_rows(out, orc, q, size, model, rows=[0])
                ok = out[3] == R.OK
                assert (out[0][ok] == out[0][0]).all() and (out[1][ok] == out[1][0]).all()
            else:
                _check_rows(out, orc, q, size, model, rows=special)
                nan = np.isnan(out[1][:len(known), 0])
                assert nan.sum() == 50
                rest = np.flatnonzero(~np.isin(known, with_vec))
                assert (out[1][rest, :out[2][0]] == -1.0).all()


def test_the_command_prints_one_list_per_user(tmp_path, capsys):
    from sparrowrecsys_b200.recforyou import main
    (tmp_path / "movies.csv").write_text("movieId,title,genres\n10,A (1995),X\n20,B (1996),X|Y\n30,C (1997),Y\n"
                                         "40,\"D, The (1998)\",Y\n")
    (tmp_path / "ratings.csv").write_text("userId,movieId,rating,timestamp\n1,10,4.0,1\n1,20,5.0,2\n2,30,3.5,3\n"
                                          "3,99,1.0,4\n")
    (tmp_path / "emb.csv").write_text("10:1 0\n20:0 1\n40:1 1\n")
    (tmp_path / "uemb.csv").write_text("1:1 0\n3:0 0\n9:1 1\n")
    args = [str(tmp_path / "movies.csv"), str(tmp_path / "ratings.csv"), "--emb", str(tmp_path / "emb.csv"),
            "--user-emb", str(tmp_path / "uemb.csv"), "--size", "3"]
    assert main(args + ["--all"]) == 0
    out = capsys.readouterr().out.splitlines()
    # averages 10: 4, 20: 5, 30: 3.5, 40: 0 -> candidates 20, 10, 30, 40
    assert out == ["1\t10:1 40:0.70710678118654746 20:0",       # user 1 = (1, 0)
                   "2\t10:-1 20:-1 30:-1",                       # no vector: all -1, by id
                   "3\t10:nan 20:nan 40:nan"]                    # a zero vector
    assert main(args + ["--user", "7", "--model", "default"]) == 0
    assert capsys.readouterr().out == "7\t(unknown user)\n"
    assert main(args + ["--user", "2", "--model", "default"]) == 0
    assert capsys.readouterr().out == "2\t20:4 10:3 30:2\n"
