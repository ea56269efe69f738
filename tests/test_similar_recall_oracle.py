"""CPU tests of the multi-channel and embedding recall oracle (oracle/similar_recall.py, a restatement of
SimilarMovieProcess.multipleRetrievalCandidates / retrievalCandidatesByEmbedding and DataManager.getMovies) on
hand-worked catalogues, of the front end's release-year rule, and of the new entry points' argument checks, which
need no device."""
import numpy as np
import pytest

from oracle import similar_movies as S
from oracle import similar_recall as R


def _cat(movies, ratings=(), emb=None):
    """movies: [(id, [genres], year)] in load order; ratings: [(movie id, score)]; emb: {id: vector}."""
    rm = [m for m, _ in ratings]
    rs = np.array([s for _, s in ratings], np.float32)
    e = (None, None) if emb is None else (list(emb), np.array(list(emb.values()), np.float32))
    return R.RecallCatalogue([m for m, _, _ in movies], [g for _, g, _ in movies], rm, rs, *e,
                             release_year=[y for _, _, y in movies])


# ---- java.util.HashMap<Integer, _> iteration order ---------------------------------------------------------------


def _order(ids):
    hm, cap = R.hashmap_order(ids)
    return [ids[i] for i in hm], cap


def test_hashmap_buckets_wrap_past_the_capacity_and_keep_load_order_within_one():
    # at 16 buckets 21 and 5 share bucket 5 (load order: 21 first), 16 is bucket 0, 31 bucket 15
    assert _order([21, 31, 5, 16, 3]) == ([16, 3, 21, 5, 31], 16)


def test_hashmap_spreads_ids_past_65536():
    # hash = id ^ (id >>> 16): 65536 -> 65537 (bucket 1, before 1 in load order), 65537 -> 65536 (bucket 0),
    # 131074 -> 131072 (bucket 0)
    assert _order([65536, 2, 65537, 131074, 1]) == ([65537, 131074, 65536, 1, 2], 16)


@pytest.mark.parametrize("n, cap", [(12, 16), (13, 32), (24, 32), (25, 64), (768, 1024), (769, 2048)])
def test_hashmap_capacity_around_a_resize(n, cap):
    ids = list(range(1000, 1000 + n))
    order, c = _order(ids)
    assert c == cap and sorted(order) == ids
    assert order == sorted(ids, key=lambda i: ((i ^ (i >> 16)) & (cap - 1), ids.index(i)))


def test_hashmap_at_twelve_and_thirteen_entries():
    ids = [3, 19, 35, 51, 1, 2, 4, 5, 6, 7, 8, 9, 10]           # 3, 19, 35, 51 share bucket 3 of 16
    assert _order(ids[:12])[0] == [1, 2, 3, 19, 35, 51, 4, 5, 6, 7, 8, 9]
    # the 13th put doubles the table: 19 and 51 move to bucket 19, behind every bucket below it
    assert _order(ids)[0] == [1, 2, 3, 35, 4, 5, 6, 7, 8, 9, 10, 19, 51]


def test_treeify_bin_resizes_a_short_table_and_rejects_a_long_one():
    ids = [64 * k for k in range(1, 10)]                        # nine in bucket 0 of 16: a resize to 32, not a tree
    assert _order(ids) == (ids, 32)
    assert R.hashmap_order(ids + [640])[1] == 64                # a tenth at 32 buckets: 64
    with pytest.raises(R.TreeifiedBin):
        R.hashmap_order(ids + [640, 704])                       # an eleventh at 64 buckets: a tree
    with pytest.raises(R.TreeifiedBin):
        R.hashmap_order(list(range(1, 61)) + [1024 * k for k in range(1, 10)])


# ---- parseReleaseYear ------------------------------------------------------------------------------------------


@pytest.mark.parametrize("title, dm, spark", [
    ("Toy Story (1995)", 1995, 1995),
    ("  Heat (1995)  ", 1995, None),            # Spark's substring bounds use the untrimmed length: it throws
    ("Up (2009) ", 2009, None),
    ("(1995)", 1995, 1995),
    ("1995)", 0, 1990),                          # shorter than 6: DataManager 0, Spark 1990
    ("", 0, 1990),
    ("Jaws (19x5)", 0, None),                    # not an int: DataManager 0, Spark throws
    ("Neg (-123)", -123, -123),
    ("Pos (+123)", 123, 123),
    ("Minus one (-001)", 0, -1),                 # parseReleaseYear's -1 means "no year": 0
    ("Untitled", 0, None),
    ("Digits 12345", 1234, 1234),
])
def test_release_year_rules(title, dm, spark):
    from sparrowrecsys_b200.featureeng import release_year
    from sparrowrecsys_b200.similar import data_manager_release_year
    assert R.parse_release_year(title) == dm == data_manager_release_year(title)
    if spark is None:
        with pytest.raises(ValueError):
            release_year(title)
    else:
        assert release_year(title) == spark


def test_release_year_counts_utf16_units():
    from sparrowrecsys_b200.similar import data_manager_release_year
    t = "\U0001F3AC (1999)"                      # one code point, two UTF-16 units, before the year
    assert R.parse_release_year(t) == data_manager_release_year(t) == 1999
    assert R.parse_release_year("\U0001F3AC1)") == data_manager_release_year("\U0001F3AC1)") == 0


# ---- getMovies and multi-channel recall ------------------------------------------------------------------------


def test_get_movies_ties_go_by_hashmap_order_across_the_100_cut():
    # 120 movies: ids 1000 .. 1119 loaded in reverse; every rating and year tied
    movies = [(i, ["A"], 2000) for i in range(1119, 999, -1)]
    c = _cat(movies)
    by_hash = [c.ids[s] for s in R.hashmap_order(c.ids)[0]]
    assert by_hash != [m for m, _, _ in movies] and by_hash != sorted(by_hash, reverse=True)
    assert [c.ids[s] for s in c.get_movies(100, "rating")] == by_hash[:100]
    assert [c.ids[s] for s in c.get_movies(100, "releaseYear")] == by_hash[:100]
    # a higher year or rating goes first whatever its bucket
    movies[-1] = (1000, ["A"], 2001)
    c = _cat(movies, [(1119, 4.0)])
    assert c.ids[c.get_movies(1, "releaseYear")[0]] == 1000 and c.ids[c.get_movies(1, "rating")[0]] == 1119


def test_year_order_is_integer_compare_descending():
    c = _cat([(1, ["A"], 0), (2, ["A"], -5), (3, ["A"], 1999), (4, ["A"], 2010), (5, ["A"], 1999)])
    assert [c.ids[s] for s in c.get_movies(10, "releaseYear")] == [4, 3, 5, 1, 2]


def test_the_pool_cut_at_10000_under_ties():
    ids = list(range(1, 10_101))
    c = _cat([(i, ["A"], 0) for i in ids], [(i, 3.0) for i in ids[:50]])
    pool = c.get_movies(R.POOL, "rating")
    assert len(pool) == R.POOL and [c.ids[s] for s in pool[:50]] == sorted(ids[:50])   # rated first, then buckets
    rest = [c.ids[s] for s in R.hashmap_order(c.ids)[0] if c.ids[s] > 50]
    assert [c.ids[s] for s in pool[50:]] == rest[:R.POOL - 50]


SMALL = [(1, ["A", "B"], 1995), (2, ["A"], 2001), (3, ["B"], 1990), (4, ["A", "B"], 0), (5, ["C"], 1980),
         (6, [], 1999)]
SMALL_R = [(1, 4.0), (2, 3.0), (3, 3.5), (5, 5.0)]


def test_multiple_candidates_exclude_the_query_and_add_the_global_lists():
    c = _cat(SMALL, SMALL_R)
    assert sorted(c.ids[s] for s in c.multiple_candidates(c.slot[1])) == [2, 3, 4, 5, 6]
    ids, scores, st = c.rec_list(1, 10, "default", "multiple")
    assert st == S.OK and 1 not in ids and sorted(ids) == [2, 3, 4, 5, 6]
    want = sorted(((c.similar_score(0, c.slot[i]), i) for i in [2, 3, 4, 5, 6]), key=lambda x: (-x[0], x[1]))
    assert ids == [i for _, i in want] and scores == [s for s, _ in want]


def test_a_query_with_no_genres_gets_the_two_global_lists():
    c = _cat(SMALL, SMALL_R)
    assert c.rec_list(6, 10, "default") == ([], [], S.OK)                    # genre candidates: none
    ids, scores, st = c.rec_list(6, 10, "default", "multiple")
    assert st == S.OK and sorted(ids) == [1, 2, 3, 4, 5]
    assert scores[ids.index(5)] == 0 / (0 + 1) / 2 * 0.7 + 5.0 / 5 * 0.3


def test_multiple_takes_each_genres_first_20():
    movies = [(i, ["X"], 0) for i in range(1, 131)] + [(500, ["X"], 0), (501, ["Y"], 0)]
    ratings = [(i, 1.0 + (i % 4)) for i in range(1, 131)]
    c = _cat(movies, ratings)
    genre20 = set(c.movies_by_genre("X", 20))
    glob = set(c.get_movies(100, "rating")) | set(c.get_movies(100, "releaseYear"))
    assert set(c.multiple_candidates(c.slot[500])) == (genre20 | glob) - {c.slot[500]}


def test_the_unknown_movie_and_a_query_without_a_vector():
    c = _cat(SMALL, SMALL_R, {1: [1, 0], 2: [1, 1]})
    assert c.rec_list(99, 5, "default", "multiple") == ([], [], S.UNKNOWN_MOVIE)
    assert c.rec_list(3, 5, "emb", "multiple") == ([], [], S.NO_EMBEDDING)
    assert c.embedding_recall(99, 5) == ([], [], S.UNKNOWN_MOVIE)
    assert c.embedding_recall(3, 5) == ([], [], S.NO_EMBEDDING)
    with pytest.raises(ValueError):
        c.rec_list(1, 5, "default", "both")


# ---- embedding recall ------------------------------------------------------------------------------------------


def test_embedding_recall_is_ascending_with_the_query_inside():
    emb = {1: [1, 0], 2: [1, 1], 3: [0, 0], 4: [-1, 0], 5: [0, 1]}            # 3 is a zero vector: NaN
    c = _cat(SMALL, SMALL_R, emb)
    ids, scores, st = c.embedding_recall(1, 10)
    # -1: 6 (no vector) and 4 (opposite), tied, by id; then 5 (0), 2, the query itself (1.0), and NaN last
    assert st == S.OK and ids == [4, 6, 5, 2, 1, 3]
    assert scores[:3] == [-1.0, -1.0, 0.0] and scores[3] == S.java_cosine([1, 0], [1, 1]) and scores[4] == 1.0
    assert np.isnan(scores[5])
    assert c.embedding_recall(1, 2)[0] == [4, 6]
    ids, scores, _ = c.embedding_recall(3, 10)                                  # a zero query: NaN but the -1
    assert ids == [6, 1, 2, 3, 4, 5] and scores[0] == -1.0 and all(np.isnan(scores[1:]))


# ---- argument checks before any device call ---------------------------------------------------------------------


def _lib():
    from sparrowrecsys_b200 import _lib as L
    return L, L.load()


def _out(n, size):
    return [np.zeros(n * max(size, 1), np.int32), np.zeros(n * max(size, 1), np.float64), np.zeros(n, np.int32),
            np.zeros(n, np.int32)]


@pytest.mark.parametrize("candidates, size, model, n, word", [
    (2, 5, 0, 1, "candidate source"), (-1, 5, 0, 1, "candidate source"), (1, 0, 0, 1, "size"),
    (1, 5, 3, 1, "model"), (1, 5, 0, -1, "n_queries"), (0, 5, 0, 1, "null catalog"), (1, 5, 1, 1, "null catalog")])
def test_candidates_call_rejections(candidates, size, model, n, word):
    L, lib = _lib()
    q = np.zeros(1, np.int32)
    p = lambda x: x.ctypes.data
    rc = lib.srs_similar_movies_candidates_host(None, candidates, p(q), n, size, model, *map(p, _out(1, size)))
    assert rc == L.SRS_ERR_INVALID and word in lib.srs_last_error().decode()


@pytest.mark.parametrize("size, n, word", [(0, 1, "size"), (-2, 1, "size"), (5, -1, "n_queries"),
                                           (5, 1, "null catalog")])
def test_embedding_recall_rejections(size, n, word):
    L, lib = _lib()
    q = np.zeros(1, np.int32)
    p = lambda x: x.ctypes.data
    assert lib.srs_similar_embedding_recall_host(None, p(q), n, size, *map(p, _out(1, size))) == L.SRS_ERR_INVALID
    assert word in lib.srs_last_error().decode()


def test_create_ex_rejects_as_create_does():
    L, lib = _lib()
    import ctypes as C
    a = lambda x, t: np.ascontiguousarray(x, t)
    ids, off, genre, year = a([7, 7], np.int32), a([0, 1, 2], np.int32), a([0, 1], np.int32), a([1995, 2000], np.int32)
    rm, rs = a([7], np.int32), a([3.0], np.float32)
    h = C.c_void_p()
    p = lambda x: x.ctypes.data
    rc = lib.srs_similar_catalog_create_ex_host(p(ids), 2, p(off), p(genre), 2, p(rm), p(rs), 1, None, None, 0, 0,
                                                p(year), 0, C.byref(h))
    assert rc == L.SRS_ERR_INVALID and not h.value and "twice" in lib.srs_last_error().decode()


def test_front_end_rejects_before_the_device():
    from sparrowrecsys_b200.similar import SimilarMovies
    movies = {"movieId": np.array([1, 2], np.int32), "genres": ["Drama", "Comedy"], "title": ["A (1995)"]}
    ratings = {"movieId": np.array([1], np.int32), "rating": np.array([3.0])}
    with pytest.raises(ValueError, match="titles"):
        SimilarMovies(movies, ratings)
