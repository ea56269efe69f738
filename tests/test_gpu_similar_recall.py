"""Multi-channel and embedding recall on the device (`SimilarMovies.recommend(..., candidates="multiple")`,
`SimilarMovies.retrieve_by_embedding`, csrc/similar.cu) against the oracle (oracle/similar_recall.py): the
reference's 982 movies with the shipped vectors, a synthetic ML-20M-sized catalogue whose HashMap order is not id
order, with tied years and ratings, vectorless and zero-vector movies, unknown and repeated queries, a table grown
by treeifyBin's resizes, a treeified one, repeat calls, and the genre candidates left as they were.  Every score is
checked bit for bit: cosines against the oracle summing in the device's lane order (`warp_cosine_many`)."""
import os

import numpy as np
import pytest

from oracle import similar_movies as S
from oracle import similar_recall as R
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200.ranking import load_embeddings_csv
from sparrowrecsys_b200.similar import SimilarMovies, data_manager_release_year, genre_lists
from test_gpu_similar import score_bits

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _oracle(movies, ratings, emb):
    return R.RecallCatalogue(movies["movieId"], genre_lists(list(movies["genres"])), ratings["movieId"],
                             np.asarray(ratings["rating"], np.float32), *(emb if emb is not None else (None, None)),
                             release_year=[data_manager_release_year(t) for t in movies["title"]],
                             cosine=S.warp_cosine_many)


def _same_list(got_ids, got_scores, want_ids, want_scores, what):
    assert got_ids.tolist() == want_ids, what
    assert np.ascontiguousarray(got_scores).tobytes() == score_bits(want_scores), what


def _check_multiple(dev, orc, queries, size, model):
    ids, scores, count, status = dev.recommend_arrays(queries, size, model, "multiple")
    for q, mid in enumerate(np.asarray(queries).tolist()):
        oi, osc, ost = orc.rec_list(mid, size, model, "multiple")
        assert status[q] == ost and count[q] == len(oi), (mid, status[q], ost, count[q], len(oi))
        _same_list(ids[q, :count[q]], scores[q, :count[q]], oi, osc, (mid, model, size))
        assert not ids[q, count[q]:].any() and not scores[q, count[q]:].any()
    return ids, scores, count, status


def _check_recall(dev, orc, queries, size, cache):
    ids, scores, count, status = dev.retrieve_by_embedding_arrays(queries, size)
    for q, mid in enumerate(np.asarray(queries).tolist()):
        if mid not in cache:
            cache[mid] = orc.embedding_recall(mid, R.POOL)
        oi, osc, ost = cache[mid]
        oi, osc = oi[:size], osc[:size]
        assert status[q] == ost and count[q] == len(oi), (mid, status[q], ost, count[q], len(oi))
        _same_list(ids[q, :count[q]], scores[q, :count[q]], oi, osc, (mid, size))
        assert not ids[q, count[q]:].any() and not scores[q, count[q]:].any()
    return ids, scores, count, status


@pytest.fixture(scope="module")
def reference():
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    r = np.load(os.path.join(GOLDEN, "featureeng_ratings.npz"))
    movies = {"movieId": m["movieId"].astype(np.int32), "genres": [str(g) for g in m["genres"]],
              "title": [str(t) for t in m["title"]]}
    ratings = {"movieId": r["movieId"].astype(np.int32), "rating": r["half"].astype(np.float64) / 2}
    emb = load_embeddings_csv(os.path.join(GOLDEN, "item2vecEmb.csv"))
    assert len(movies["movieId"]) == 982
    dev = SimilarMovies(movies, ratings, emb)
    yield movies, ratings, emb, dev, _oracle(movies, ratings, emb), {}
    dev.close()


@pytest.mark.parametrize("model", ["default", "emb"])
@pytest.mark.parametrize("size", [10, 2000])
def test_reference_multiple_candidates(reference, model, size):
    movies, _, _, dev, orc, _ = reference
    _, _, count, status = _check_multiple(dev, orc, movies["movieId"], size, model)
    if model == "default":
        assert (status == S.OK).all() and count.min() >= (10 if size == 10 else 100)


@pytest.mark.parametrize("size", [10, 2000])
def test_reference_embedding_recall(reference, size):
    movies, _, _, dev, orc, cache = reference
    ids, scores, count, status = _check_recall(dev, orc, movies["movieId"], size, cache)
    ok = status == S.OK
    assert (status[~ok] == S.NO_EMBEDDING).all() and ok.sum() == len(orc.emb)
    assert (count[ok] == min(size, 982)).all()
    if size == 2000:               # the query is in its own pool, and the -1s of the vectorless movies come first
        for q in np.flatnonzero(ok)[:50]:
            assert movies["movieId"][q] in ids[q, :count[q]].tolist()
            assert (scores[q, :982 - len(orc.emb)] == -1.0).all()


def test_reference_default_candidates_are_unchanged(reference):
    movies, ratings, emb, dev, _, _ = reference
    without_titles = {"movieId": movies["movieId"], "genres": movies["genres"]}
    with SimilarMovies(without_titles, ratings, emb) as old:
        for model in ("default", "emb"):
            a = dev.recommend_arrays(movies["movieId"], 50, model)
            b = old.recommend_arrays(movies["movieId"], 50, model)
            c = dev.recommend_arrays(movies["movieId"], 50, model, "genre")
            assert all(x.tobytes() == y.tobytes() == z.tobytes() for x, y, z in zip(a, b, c))
        with pytest.raises(ValueError, match="release years"):
            old.recommend(movies["movieId"][:3], 10, "default", "multiple")
        q = np.ascontiguousarray(movies["movieId"][:3], np.int32)
        out = [np.zeros(30, np.int32), np.zeros(30, np.float64), np.zeros(3, np.int32), np.zeros(3, np.int32)]
        p = lambda a: a.ctypes.data
        assert _lib.load().srs_similar_movies_candidates_host(old._h, _lib.SRS_SIMILAR_CANDIDATES_MULTIPLE, p(q), 3,
                                                              10, 0, *map(p, out)) == _lib.SRS_ERR_INVALID
        assert old.retrieve_by_embedding(q, 5)[0].status == S.OK      # embedding recall needs no years


def test_a_second_call_gives_the_same_bits(reference):
    movies, _, _, dev, _, _ = reference
    for call in (lambda: dev.recommend_arrays(movies["movieId"], 300, "default", "multiple"),
                 lambda: dev.recommend_arrays(movies["movieId"], 300, "emb", "multiple"),
                 lambda: dev.retrieve_by_embedding_arrays(movies["movieId"], 2000)):
        a, b = call(), call()
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def synthetic_catalogue(seed=11, n=27_278, max_id=131_262, dim=16):
    """ML-20M-sized: ids up to max_id in a shuffled load order (so HashMap order is neither id nor load order), 1-4
    of 20 genres, ratings from three values with most movies unrated or rated once (ties in the average across
    every cut), years from a dozen values or unparsable (0), 16-dim vectors for 80 % and a few zero vectors."""
    rng = np.random.default_rng(seed)
    ids = rng.permutation(np.arange(1, max_id, dtype=np.int32))[:n]
    ids[-1] = max_id
    genres = ["|".join("G%d" % g for g in rng.choice(20, rng.integers(1, 5), replace=False)) for _ in range(n)]
    years = rng.integers(1990, 2002, n)
    titles = ["Movie %d (%d)" % (i, y) if rng.random() > 0.05 else "Untitled" for i, y in zip(ids, years)]
    rated = rng.random(n) < 0.6
    rm = ids[rated][rng.integers(0, int(rated.sum()), 40_000)]
    rs = rng.choice([3.0, 4.0, 5.0], rm.shape[0])
    has = rng.random(n) < 0.8
    vec = rng.standard_normal((int(has.sum()), dim)).astype(np.float32)
    vec[:3] = 0.0                                                          # cosines of 0 / 0: NaN
    movies = {"movieId": ids, "genres": genres, "title": titles}
    return movies, {"movieId": rm.astype(np.int32), "rating": rs}, (ids[has], vec)


@pytest.fixture(scope="module")
def synthetic():
    movies, ratings, emb = synthetic_catalogue()
    dev = SimilarMovies(movies, ratings, emb)
    orc = _oracle(movies, ratings, emb)
    ids = movies["movieId"]
    rng = np.random.default_rng(5)
    vectorless = ids[~np.isin(ids, emb[0])][:5]
    q = np.concatenate([ids[rng.integers(0, len(ids), 120)], emb[0][:3], vectorless, [0, -5, 10 ** 8, 131_263],
                        ids[:3], ids[:3], [ids[orc.get_movies(1, "rating")[0]]]]).astype(np.int32)
    yield movies, dev, orc, q, vectorless
    dev.close()


def test_synthetic_catalogue_orders(synthetic):
    movies, _, orc, _, _ = synthetic
    hm, cap = R.hashmap_order(orc.ids)
    assert cap == 65536 and hm != sorted(hm)
    pool = orc.get_movies(R.POOL, "rating")
    assert orc.avg[pool[-1]] == orc.avg[orc.get_movies(R.POOL + 1, "rating")[-1]]        # ties across the cut
    top = orc.get_movies(100, "releaseYear")
    assert orc.year[top[-1]] == orc.year[orc.get_movies(101, "releaseYear")[-1]] == 2001


def _vectorless(orc, queries):
    return sum(1 for mid in np.asarray(queries).tolist() if mid in orc.slot and orc.slot[mid] not in orc.emb)


@pytest.mark.parametrize("model", ["default", "emb"])
def test_synthetic_multiple_candidates(synthetic, model):
    _, dev, orc, q, _ = synthetic
    for size in (7, 500):
        _, _, _, status = _check_multiple(dev, orc, q, size, model)
        assert (status == S.UNKNOWN_MOVIE).sum() == 4
        assert (status == S.NO_EMBEDDING).sum() == (_vectorless(orc, q) if model == "emb" else 0)


def test_synthetic_embedding_recall(synthetic):
    _, dev, orc, q, vectorless = synthetic
    assert _vectorless(orc, q) >= len(vectorless)
    cache = {}
    for size in (10, 2000):
        _, scores, count, status = _check_recall(dev, orc, q, size, cache)
        assert (status == S.UNKNOWN_MOVIE).sum() == 4 and (status == S.NO_EMBEDDING).sum() == _vectorless(orc, q)
    zero = q[120:123]                                                       # queries with a zero vector: all NaN
    _, fs, fc, st = dev.retrieve_by_embedding_arrays(zero, 10_000)
    assert (st == S.OK).all() and (fc == R.POOL).all() and np.isnan(fs[:, -1]).all()
    assert not np.isnan(fs[:, 0]).any()                                     # the -1s of vectorless movies first


def _flat_catalogue(ids):
    """Unrated movies of one genre and one year: getMovies' orders are movieMap's iteration order."""
    n = len(ids)
    return ({"movieId": np.asarray(ids, np.int32), "genres": ["A"] * n, "title": ["M (2000)"] * n},
            {"movieId": np.zeros(0, np.int32), "rating": np.zeros(0)})


def test_treeify_resizes_and_a_treeified_table():
    # ten ids in bucket 0 while the table is short: treeifyBin doubles it twice instead of building a tree
    ids = [64 * k for k in range(1, 11)] + [x for x in range(70_001, 80_000) if (x ^ x >> 16) & 63][:140]
    assert R.hashmap_order(ids)[1] == 256
    movies, ratings = _flat_catalogue(ids)
    orc = _oracle(movies, ratings, None)
    with SimilarMovies(movies, ratings) as dev:
        _check_multiple(dev, orc, [ids[0], ids[-1], 5], 150, "default")
    # a ninth id in one bucket of a 128-bucket table: Java makes the bin a tree
    ids = list(range(1, 61)) + [1024 * k for k in range(1, 10)]
    with pytest.raises(R.TreeifiedBin):
        R.hashmap_order(ids)
    movies, ratings = _flat_catalogue(ids)
    with SimilarMovies(movies, ratings) as dev:
        assert dev.recommend(ids[:2], 5, "default")[0].status == S.OK       # the genre candidates still work
        for call in (lambda: dev.recommend(ids[:2], 5, "default", "multiple"),
                     lambda: dev.retrieve_by_embedding(ids[:2], 5)):
            with pytest.raises(_lib.SrsInvalidError, match="treeified"):
                call()
