"""CPU tests of the similar-movies oracle (oracle/similar_movies.py, a restatement of SimilarMovieProcess.getRecList)
on hand-worked catalogues, and of the library's and the front end's argument checks, which need no device."""
import ctypes as C

import numpy as np
import pytest

from oracle import similar_movies as S


def _cat(movies, ratings=(), emb=None):
    """movies: [(id, [genres])] in load order; ratings: [(movie id, score)] in file order; emb: {id: vector}."""
    ids = [m for m, _ in movies]
    rm = [m for m, _ in ratings]
    rs = np.array([s for _, s in ratings], np.float32)
    if emb is None:
        return S.Catalogue(ids, [g for _, g in movies], rm, rs)
    return S.Catalogue(ids, [g for _, g in movies], rm, rs, list(emb), np.array(list(emb.values()), np.float32))


SMALL = [(1, ["A", "B"]), (2, ["A"]), (3, ["B"]), (4, ["A", "B"]), (5, ["C"]),
         (6, ["(no genres listed)"]), (7, ["(no genres listed)"]), (8, [])]
SMALL_R = [(1, 4.0), (2, 3.0), (3, 3.0), (5, 5.0), (6, 2.0), (7, 2.0)]


def test_ties_in_average_rating_keep_load_order():
    movies = [(10 + i, ["X"]) for i in range(150)] + [(500, ["X"])]
    ratings = [(10 + i, 3.0) for i in range(150)] + [(500, 4.0)]
    c = _cat(movies, ratings)
    top = [c.ids[m] for m in c.movies_by_genre("X")]
    assert top == [500] + [10 + i for i in range(99)]


def test_a_candidate_in_several_genres_is_counted_once_and_the_query_is_excluded():
    c = _cat(SMALL, SMALL_R)
    ids, scores, st = c.rec_list(1, 50, "default")
    assert st == S.OK and sorted(ids) == [2, 3, 4] and len(ids) == 3
    assert 1 not in ids


def test_a_genre_with_fewer_than_100_movies():
    c = _cat(SMALL, SMALL_R)
    assert [c.ids[m] for m in c.movies_by_genre("A")] == [1, 2, 4]
    assert [c.ids[m] for m in c.movies_by_genre("C")] == [5]


def test_an_unrated_movie_averages_zero():
    c = _cat(SMALL, SMALL_R)
    assert c.avg[c.slot[4]] == 0.0
    ids, scores, _ = c.rec_list(1, 50, "default")
    # movie 4 shares both genres: 2 / (2 + 2) / 2 * 0.7 + 0 / 5 * 0.3
    assert scores[ids.index(4)] == 2 / 4 / 2 * 0.7 + 0.0 / 5 * 0.3


def test_hand_worked_default_scores_and_order():
    c = _cat(SMALL, SMALL_R)
    ids, scores, _ = c.rec_list(1, 50, "default")
    s2 = 1 / 3 / 2 * 0.7 + 3.0 / 5 * 0.3        # one shared genre of 2 + 1
    s4 = 2 / 4 / 2 * 0.7 + 0.0
    assert ids == [2, 3, 4] and scores == [s2, s2, s4]      # 2 and 3 tie: by id


def test_no_genres_listed_is_an_ordinary_genre_and_no_genres_gives_nothing():
    c = _cat(SMALL, SMALL_R)
    ids, scores, st = c.rec_list(6, 10, "default")
    assert ids == [7] and scores == [1 / 2 / 2 * 0.7 + 2.0 / 5 * 0.3]
    assert c.rec_list(8, 10, "default") == ([], [], S.OK)


def test_a_tied_final_score_goes_by_movie_id_not_load_order():
    c = _cat([(21, ["D"]), (20, ["D"]), (22, ["D"]), (19, ["D"])], [(21, 3.0), (20, 3.0), (19, 1.0)])
    ids, scores, _ = c.rec_list(22, 10, "default")
    assert ids == [20, 21, 19] and scores[0] == scores[1]


def test_emb_with_missing_vectors():
    emb = {1: [1, 0], 2: [1, 1], 4: [0, 1]}
    c = _cat(SMALL, SMALL_R, emb)
    assert c.rec_list(3, 10, "emb") == ([], [], S.NO_EMBEDDING)        # the Java throws on the query
    ids, scores, st = c.rec_list(1, 10, "emb")
    # candidate 3 has no vector: Embedding.calculateSimilarity(null) is -1
    assert st == S.OK and ids == [2, 4, 3]
    assert scores == [S.java_cosine([1, 0], [1, 1]), 0.0, -1.0]
    # the default ranker does not need vectors
    assert c.rec_list(3, 10, "default")[2] == S.OK


def test_the_unknown_movie_gives_an_empty_list():
    c = _cat(SMALL, SMALL_R)
    assert c.rec_list(999, 10, "default") == ([], [], S.UNKNOWN_MOVIE)
    assert c.rec_list(999, 10, "emb") == ([], [], S.UNKNOWN_MOVIE)


def test_the_size_cut():
    c = _cat(SMALL, SMALL_R)
    assert c.rec_list(1, 2, "default")[0] == [2, 3]


RUNNING = [1.5, 5.0, 4.0, 1.0, 3.5, 4.0, 1.0, 1.0, 2.0, 0.5, 2.5, 2.5, 3.5, 3.0, 2.5, 1.5, 3.0, 2.5, 4.5, 3.5, 4.0,
           3.0, 2.0, 1.5, 2.5, 3.0, 2.0]


def test_the_running_mean_is_not_the_mean():
    a = S.running_mean(RUNNING)
    assert a != np.mean(RUNNING)
    assert abs(np.frexp(a)[0] - np.frexp(np.mean(RUNNING))[0]) * 2 ** 53 == 1      # one unit in the last place
    assert a == float.fromhex("0x1.4e38e38e38e3ap+1")
    c = _cat([(1, ["A"]), (2, ["A"])], [(2, s) for s in RUNNING])
    assert c.avg[1] == a


def test_double_compare_order_of_averages():
    # NaN first (Double.compare), ties in load order.  A single -0.0 rating averages to +0.0, (0.0 * 0 + -0.0) / 1,
    # so it ties with the unrated movie 2
    c = _cat([(1, ["A"]), (2, ["A"]), (3, ["A"]), (4, ["A"])], [(1, -0.0), (3, float("nan")), (4, -1.0)])
    assert np.copysign(1.0, c.avg[0]) == 1.0
    assert [c.ids[m] for m in c.movies_by_genre("A")] == [3, 1, 2, 4]


def test_java_cosine_many_matches_the_literal_loop():
    rng = np.random.default_rng(0)
    q = rng.standard_normal(10).astype(np.float32)
    M = rng.standard_normal((20, 10)).astype(np.float32)
    assert np.array_equal(S.java_cosine_many(q, M), [S.java_cosine(q, m) for m in M])


# ---- the front end's parsing ---------------------------------------------------------------------------------


def test_genre_lists_and_data_manager_rows(tmp_path):
    from sparrowrecsys_b200.similar import data_manager_rows, genre_lists, java_split
    assert java_split("a|b||", "|") == ["a", "b"] and java_split("", ",") == [""] and java_split("|a", "|") == ["", "a"]
    assert genre_lists(["Drama|Comedy", "(no genres listed)", " ", "|"]) == [["Drama", "Comedy"],
                                                                            ["(no genres listed)"], [], []]
    p = tmp_path / "movies.csv"
    p.write_text('movieId,title,genres\n1,Toy Story (1995),Animation\n2,"President, The (1995)",Drama\n'
                 '3,Heat (1995),\n4,Up (2009),Comedy\n')
    assert data_manager_rows(str(p)).tolist() == [1, 4]


# ---- argument checks before any device call ---------------------------------------------------------------------


def _lib():
    from sparrowrecsys_b200 import _lib as L
    return L, L.load()


def _create(lib, ids, off, genre, n_genres, rm=(1,), rs=(3.0,), n_r=None, eid=(1,), emb=(0.5,), n_emb=0, dim=0):
    a = lambda x, t: np.ascontiguousarray(x, t)
    ids, off, genre = a(ids, np.int32), a(off, np.int32), a(genre or [0], np.int32)
    rm, rs, eid, emb = a(rm, np.int32), a(rs, np.float32), a(eid, np.int32), a(emb, np.float32)
    h = C.c_void_p()
    p = lambda x: x.ctypes.data
    rc = lib.srs_similar_catalog_create_host(p(ids), ids.shape[0], p(off), p(genre), n_genres, p(rm), p(rs),
                                             rm.shape[0] if n_r is None else n_r, p(eid), p(emb), n_emb, dim, 0,
                                             C.byref(h))
    return rc, h


@pytest.mark.parametrize("case", ["too_many_genres", "genre_out_of_range", "repeated_genre", "repeated_id",
                                  "bad_offsets", "negative_ratings", "vectors_without_width"])
def test_catalog_rejections(case):
    L, lib = _lib()
    args = dict(ids=[1, 2], off=[0, 1, 2], genre=[0, 1], n_genres=2)
    if case == "too_many_genres":
        args["n_genres"] = 65
    elif case == "genre_out_of_range":
        args["genre"] = [0, 2]
    elif case == "repeated_genre":
        args.update(off=[0, 2, 2], genre=[1, 1])
    elif case == "repeated_id":
        args["ids"] = [7, 7]
    elif case == "bad_offsets":
        args["off"] = [1, 1, 2]
    elif case == "negative_ratings":
        args["n_r"] = -1
    elif case == "vectors_without_width":
        args.update(n_emb=1, dim=0)
    rc, h = _create(lib, **args)
    assert rc == L.SRS_ERR_INVALID and not h.value
    assert lib.srs_last_error()


@pytest.mark.parametrize("size, model, n", [(0, 0, 1), (-3, 1, 1), (5, 2, 1), (5, 0, -1)])
def test_query_rejections(size, model, n):
    L, lib = _lib()
    q = np.zeros(1, np.int32)
    ids, cnt, st = np.zeros(8, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32)
    sc = np.zeros(8, np.float64)
    p = lambda x: x.ctypes.data
    assert lib.srs_similar_movies_host(None, p(q), n, size, model, p(ids), p(sc), p(cnt), p(st)) == L.SRS_ERR_INVALID
    msg = lib.srs_last_error().decode()
    assert ("size" in msg) == (size < 1) and ("model" in msg) == (size >= 1 and model == 2)


def test_front_end_rejects_before_the_device():
    from sparrowrecsys_b200 import _lib as L
    from sparrowrecsys_b200.similar import SimilarMovies
    movies = {"movieId": np.array([1, 2], np.int32), "genres": ["Drama|Drama", "Comedy"]}
    ratings = {"movieId": np.array([1], np.int32), "rating": np.array([3.0])}
    with pytest.raises(L.SrsInvalidError, match="twice"):
        SimilarMovies(movies, ratings)
    movies["genres"] = ["Drama", "Comedy"]
    with pytest.raises(ValueError, match="embeddings"):
        SimilarMovies(movies, ratings, (np.array([1, 2], np.int32), np.zeros((3, 4), np.float32)))
    movies["genres"] = ["|".join("g%d" % i for i in range(65)), "Comedy"]
    with pytest.raises(L.SrsInvalidError, match="66 genres"):          # g0 .. g64 and Comedy
        SimilarMovies(movies, ratings)
