"""Similar movies on the device (`SimilarMovies`, `srs_similar_movies_host`, csrc/similar.cu) against the oracle
(oracle/similar_movies.py): the reference's 982 movies with both rankers, a synthetic catalogue past 65 536 movies
with more than 100 tied ratings in a genre, repeated and unknown query ids, repeat calls and the rejections.  Every
score is checked bit for bit: cosines against the oracle summing in the device's lane order (`warp_cosine_many`)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import similar_movies as S
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200.ranking import load_embeddings_csv
from sparrowrecsys_b200.similar import SimilarMovies, genre_lists

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def score_bits(x):
    """The bytes of float64 scores with every NaN as the device writes it (the quiet NaN 0x7ff8000000000000)."""
    x = np.array(x, np.float64)
    x[np.isnan(x)] = np.nan
    return x.tobytes()


def _oracle(movies, ratings, emb):
    return S.Catalogue(movies["movieId"], genre_lists(list(movies["genres"])), ratings["movieId"],
                       np.asarray(ratings["rating"], np.float32), *(emb if emb is not None else (None, None)),
                       cosine=S.warp_cosine_many)


def _check(dev, orc, queries, size, model):
    ids, scores, count, status = dev.recommend_arrays(queries, size, model)
    for q, mid in enumerate(np.asarray(queries).tolist()):
        oi, osc, ost = orc.rec_list(mid, size, model)
        assert status[q] == ost, (mid, status[q], ost)
        assert count[q] == len(oi), (mid, count[q], len(oi))
        assert ids[q, :count[q]].tolist() == oi, (mid, model, size)
        assert not ids[q, count[q]:].any() and not scores[q, count[q]:].any()
        assert scores[q, :count[q]].tobytes() == score_bits(osc), (mid, model, size)
    return ids, scores, count, status


@pytest.fixture(scope="module")
def reference():
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    r = np.load(os.path.join(GOLDEN, "featureeng_ratings.npz"))
    movies = {"movieId": m["movieId"].astype(np.int32), "genres": [str(g) for g in m["genres"]]}
    ratings = {"movieId": r["movieId"].astype(np.int32), "rating": r["half"].astype(np.float64) / 2}
    emb = load_embeddings_csv(os.path.join(GOLDEN, "item2vecEmb.csv"))
    assert len(movies["movieId"]) == 982 and len(ratings["movieId"]) == 203150
    dev = SimilarMovies(movies, ratings, emb)
    yield movies, dev, _oracle(movies, ratings, emb)
    dev.close()


@pytest.mark.parametrize("model", ["default", "emb"])
@pytest.mark.parametrize("size", [10, 2000])
def test_reference_movies(reference, model, size):
    movies, dev, orc = reference
    ids, _, count, status = _check(dev, orc, movies["movieId"], size, model)
    if model == "emb":             # 101 of the 982 movies have no vector
        assert (status == S.NO_EMBEDDING).sum() == 982 - len(orc.emb)
    if size == 2000:
        assert count.max() < 2000


def test_a_second_call_gives_the_same_bits(reference):
    movies, dev, _ = reference
    for model in ("default", "emb"):
        a = dev.recommend_arrays(movies["movieId"], 50, model)
        b = dev.recommend_arrays(movies["movieId"], 50, model)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_rejections_leave_the_catalogue_usable(reference):
    movies, dev, _ = reference
    before = dev.recommend_arrays(movies["movieId"][:20], 10, "default")
    lib = _lib.load()
    q = np.ascontiguousarray(movies["movieId"][:20], np.int32)
    out = [np.zeros(200, np.int32), np.zeros(200, np.float64), np.zeros(20, np.int32), np.zeros(20, np.int32)]
    p = lambda a: a.ctypes.data
    for size, model in ((0, 0), (10, 5), (-1, 1)):
        assert lib.srs_similar_movies_host(dev._h, p(q), 20, size, model, *map(p, out)) == _lib.SRS_ERR_INVALID
    with pytest.raises(ValueError):
        dev.recommend(movies["movieId"][:20], 0, "default")
    after = dev.recommend_arrays(movies["movieId"][:20], 10, "default")
    assert all(x.tobytes() == y.tobytes() for x, y in zip(before, after))


@pytest.fixture(scope="module")
def synthetic():
    rng = np.random.default_rng(7)
    n, n_genres = 70_000, 20
    ids = rng.permutation(np.arange(1, 3 * n, dtype=np.int32))[:n]           # not in id order
    genres = []
    for i in range(n):
        k = rng.integers(1, 4)
        genres.append("|".join("G%d" % g for g in rng.choice(n_genres, k, replace=False)))
    # genre G0's first 300 movies all average exactly 4.5: more than 100 tied at the top of its list
    g0 = [i for i in range(n) if "G0" in genres[i].split("|")][:300]
    rm = [ids[i] for i in g0 for _ in range(2)]
    rs = [4.5] * len(rm)
    other = rng.integers(0, n, 1_000_000 - len(rm))
    other = other[~np.isin(other, g0)]
    rm += ids[other].tolist()
    rs += (rng.integers(1, 11, other.shape[0]) / 2).tolist()
    rm += [10 ** 8] * 5                                                     # ratings of a movie outside the catalogue
    rs += [5.0] * 5
    movies = {"movieId": ids, "genres": genres}
    ratings = {"movieId": np.array(rm, np.int32), "rating": np.array(rs)}
    has = rng.random(n) < 0.8
    emb = (ids[has], rng.standard_normal((int(has.sum()), 16)).astype(np.float32))
    dev = SimilarMovies(movies, ratings, emb)
    yield movies, dev, _oracle(movies, ratings, emb), g0
    dev.close()


def test_synthetic_catalogue_past_65536_movies(synthetic):
    movies, dev, orc, g0 = synthetic
    ids = movies["movieId"]
    top = orc.movies_by_genre("G0")
    assert [orc.avg[m] for m in top] == [4.5] * 100 and top == sorted(top)     # tied, in load order
    rng = np.random.default_rng(3)
    q = np.concatenate([ids[g0[:5]], ids[rng.integers(0, len(ids), 300)], ids[-3:], ids[:3],
                        [0, -5, 10 ** 8, 2 ** 31 - 1], ids[g0[:5]]]).astype(np.int32)
    for model in ("default", "emb"):
        for size in (7, 500):
            _, _, _, status = _check(dev, orc, q, size, model)
            assert (status == S.UNKNOWN_MOVIE).sum() >= 3
