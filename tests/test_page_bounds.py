"""The similar-movies and recommended-for-you pages at their bounds, on the CPU: the oracles' genreless score, the
device's lane-order cosine (`warp_cosine_many`) against the Java's index order, the "nerualcf" kernels'
instantiations, and hand-worked answers on the catalogues that tests/test_gpu_page_bounds.py runs on the device.

The catalogue builders here are shared with that file:
* `genre_catalogue(kind)`: the sort widths of sim_query_kernel - a largest candidate list of 1, 32, 33, 256, 257
  and 6 400 entries (np 32, 32, 64, 256, 512 and 8 192), genres of exactly 99, 100 and 101 movies, 64 genres;
* `small_multi_catalogue()`: fewer than 100 movies (both global lists hold all of them), genreless movies;
* `flat_catalogue(n, dim)`: n movies, ratings tied across every cut, for the recall pools and RecForYou's sort;
* `width_catalogue(dim)`: vectors of `dim` with duplicates and pairs one ulp apart in one element.
"""
import os
import re

import numpy as np
import pytest

from oracle import recforyou as RF
from oracle import similar_movies as S
from oracle import similar_recall as R
from oracle.recforyou_features import history_positions, read_history_keys
from sparrowrecsys_b200.similar import data_manager_release_year, genre_lists
from sparrowrecsys_b200.spec import default_spec, history_keys

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc")
WIDTHS = (1, 31, 32, 33, 64, 65, 300)


# ---- catalogues -------------------------------------------------------------------------------------------------
def _movies(genres, seed, dim, top_first=True, ids=None):
    """(movies, ratings, emb) of movies with `genres` (lists) in load order: ids 1.. (or `ids`), titles with a year
    from a dozen, one rating each from five half-star values (so averages tie across every cut) and movie 0 rated
    5.0 twice when `top_first`, `dim`-wide normal vectors for every movie."""
    rng = np.random.default_rng(seed)
    n = len(genres)
    ids = np.arange(1, n + 1, dtype=np.int32) if ids is None else np.asarray(ids, np.int32)
    titles = ["M%d (%d)" % (i, y) for i, y in zip(ids.tolist(), rng.integers(1990, 2002, n).tolist())]
    rm = ids.tolist()
    rs = rng.choice([1.0, 2.0, 3.0, 3.5, 4.0], n).tolist()
    if top_first:
        rs[0] = 5.0
        rm.append(int(ids[0]))
        rs.append(5.0)
    movies = {"movieId": ids, "genres": ["|".join(g) for g in genres], "title": titles}
    ratings = {"movieId": np.array(rm, np.int32), "rating": np.array(rs)}
    return movies, ratings, (ids, rng.standard_normal((n, dim)).astype(np.float32))


def genre_catalogue(kind, dim=33):
    """(movies, ratings, emb, queries, max_cands): `kind` is the largest candidate list, before the query leaves it.
    Movie 0 (id 1) carries every genre of the catalogue and is the best rated; `queries` holds it, one movie of each
    genre, a genreless movie and an unknown id."""
    def own(g, k):
        return [[g] for _ in range(k)]
    if kind == 1:                      # every genre one movie: no candidates at all
        genres = [["A"], ["B"], ["C"]]
    elif kind in (32, 33):             # one genre of 32 / 33
        genres = [["A"]] + own("A", kind - 1) + own("B", 3)
    elif kind == 256:                  # genres of exactly 99, 100 and 57 movies
        genres = [["A", "B", "C"]] + own("A", 98) + own("B", 99) + own("C", 56)
    elif kind == 257:                  # 100, 101 (its list keeps 100) and 57
        genres = [["A", "B", "C"]] + own("A", 99) + own("B", 100) + own("C", 56)
    elif kind == 6400:                 # 64 genres of 101 .. 104 movies; movie 1 only G63, movie 2 G0 and G63,
        all64 = ["G%d" % g for g in range(64)]            # movie 3 G40 and G63: two genre bits past 31
        genres = [all64, ["G63"], ["G0", "G63"], ["G40", "G63"]]
        for g in range(64):
            genres += own("G%d" % g, 100 + g % 3)
    else:
        raise ValueError(kind)
    genres.append([])                  # a genreless movie: no candidates under GENRE
    movies, ratings, emb = _movies(genres, kind, dim)
    if kind == 6400:                   # movies 1 .. 3 rate lowest: in no genre's top 100
        ratings["rating"][1:4] = 0.5
    ids = movies["movieId"]
    first = {}
    for m, gl in enumerate(genres[1:], 1):
        for g in gl:
            first.setdefault(g, m)
    extra = [ids[1], ids[2], ids[3]] if kind == 6400 else []
    q = [ids[0]] + extra + [ids[m] for m in sorted(set(first.values()))] + [ids[-1], 10 ** 6]
    return movies, ratings, emb, np.array(q, np.int32), kind


def small_multi_catalogue(dim=16):
    """40 movies, 10 of them genreless, so getMovies(100, ...) holds every movie; movie 0 is genreless too."""
    genres = [[]] + [[] if m % 4 == 0 else ["G%d" % (m % 3)] for m in range(1, 40)]
    return _movies(genres, 40, dim, top_first=False)


def flat_catalogue(n, dim=16, seed=0):
    """n movies of genres G0..G4 in a shuffled id order, ratings tied across every cut."""
    rng = np.random.default_rng(seed + n)
    ids = rng.permutation(np.arange(1, 3 * n + 2, dtype=np.int32))[:n]
    genres = [["G%d" % (m % 5)] for m in range(n)]
    return _movies(genres, seed + n, dim, top_first=False, ids=ids)


def width_catalogue(dim, n=300):
    """n movies with `dim`-wide vectors: rows 10..19 duplicate rows 0..9 (exact ties, ordered by id), rows 20..29
    are rows 0..9 with one element moved by one ulp, and past 33 rows 31 and 30 are `ulp_apart_pair`, in one
    genre."""
    movies, ratings, (ids, vec) = flat_catalogue(n, dim, seed=dim)
    vec[10:20] = vec[0:10]
    vec[20:30] = vec[0:10]
    k = np.arange(10) % dim
    vec[np.arange(20, 30), k] = np.nextafter(vec[np.arange(20, 30), k], np.float32(np.inf))
    if dim >= 34:                      # movies 30 and 31: a pair whose cosine the Java's order rounds apart
        vec[31], vec[30] = ulp_apart_pair(dim)
        movies["genres"][31] = movies["genres"][30]
    return movies, ratings, (ids, vec)


def recall_oracle(movies, ratings, emb, cosine=S.warp_cosine_many):
    return R.RecallCatalogue(movies["movieId"], genre_lists(list(movies["genres"])), ratings["movieId"],
                             np.asarray(ratings["rating"], np.float32), *(emb if emb is not None else (None, None)),
                             release_year=[data_manager_release_year(t) for t in movies["title"]], cosine=cosine)


# ---- the genreless pair -----------------------------------------------------------------------------------------
def _genreless():
    #            id  genres  rating
    movies = [(5, [], 4.0), (3, [], 2.0), (9, ["A"], 5.0), (7, [], 3.0), (1, ["A", "B"], 1.0)]
    return R.RecallCatalogue([m for m, _, _ in movies], [g for _, g, _ in movies], [m for m, _, _ in movies],
                             np.array([r for _, _, r in movies], np.float32), release_year=[2000] * 5)


def test_the_genreless_pair_scores_nan_and_comes_first_by_id():
    c = _genreless()
    assert np.isnan(c.similar_score(c.slot[5], c.slot[3]))
    ids, scores, st = c.rec_list(5, 10, "default", "multiple")
    assert st == S.OK and ids == [3, 7, 9, 1]            # the two NaNs first, by id; then 5.0 / 5 * 0.3 > 0.06
    assert np.isnan(scores[0]) and np.isnan(scores[1])
    assert scores[2:] == [5.0 / 5 * 0.3, 1.0 / 5 * 0.3]
    assert c.rec_list(5, 10, "default", "genre")[0] == []    # no genre, no genre candidates


def test_a_genreless_candidate_against_a_query_with_genres_is_unchanged():
    c = _genreless()
    assert c.similar_score(c.slot[9], c.slot[3]) == 0 / 1 / 2 * 0.7 + 2.0 / 5 * 0.3
    assert c.similar_score(c.slot[1], c.slot[7]) == 0 / 2 / 2 * 0.7 + 3.0 / 5 * 0.3
    assert c.similar_score(c.slot[1], c.slot[9]) == 1 / 3 / 2 * 0.7 + 5.0 / 5 * 0.3


# ---- the device's lane order against the Java's index order ---------------------------------------------------
@pytest.mark.parametrize("dim", WIDTHS)
def test_warp_cosine_against_java_order(dim):
    rng = np.random.default_rng(dim)
    q = rng.standard_normal(dim).astype(np.float32)
    C = rng.standard_normal((5000, dim)).astype(np.float32)
    w, j = S.warp_cosine_many(q, C), S.java_cosine_many(q, C)
    assert np.abs(w - j).max() <= 1e-15
    # multiples of 1/64 below 5 in magnitude: every product and every sum is exact, so the orders agree bit for bit
    Qd, Cd = np.round(q * 64) / 64, np.round(C * 64) / 64
    assert S.warp_cosine_many(Qd, Cd).tobytes() == S.java_cosine_many(Qd, Cd).tobytes()
    if dim == 1:
        assert w.tobytes() == j.tobytes()
    # the literal per-lane loop of cosine.cuh on a few rows
    for r in range(3):
        lanes = [[0.0] * 32 for _ in range(3)]
        for k in range(dim):
            a, b = q[k], C[r, k]
            for s, x in zip(lanes, (a * b, a * a, b * b)):
                s[k % 32] += float(np.float32(x))
        tot = []
        for s in lanes:
            for o in (16, 8, 4, 2, 1):
                s = [s[l] + s[l ^ o] for l in range(32)]
            tot.append(s[0])
        assert w[r] == tot[0] / (np.sqrt(tot[1]) * np.sqrt(tot[2]))
    zero = np.zeros((2, dim), np.float32)
    assert np.isnan(S.warp_cosine_many(q, zero)).all() and np.isnan(S.warp_cosine_many(zero[0], C[:4])).all()


def ulp_apart_pair(dim):
    """(q, v) whose cosine the two orders round apart (dim >= 34): q all ones, v = 1 at 0 and 2^-53 at 1 and 33.
    Java adds each 2^-53 to 1 and loses it; the device's lane 1 sums them to 2^-52 first, which 1 keeps."""
    q = np.ones(dim, np.float32)
    v = np.zeros(dim, np.float32)
    v[0], v[1], v[33] = 1.0, 2.0 ** -53, 2.0 ** -53
    return q, v


def test_the_two_orders_are_distinct_at_wide_vectors():
    for dim in (64, 65, 300):
        q, v = ulp_apart_pair(dim)
        w, j = S.warp_cosine_many(q, v[None])[0], S.java_cosine_many(q, v[None])[0]
        assert j == 1 / np.sqrt(dim) and w == (1 + 2.0 ** -52) / np.sqrt(dim) and w != j
        rng = np.random.default_rng(dim)
        q = rng.standard_normal(dim).astype(np.float32)
        C = rng.standard_normal((20000, dim)).astype(np.float32)
        assert (S.warp_cosine_many(q, C) != S.java_cosine_many(q, C)).any(), dim


def test_the_width_catalogues_carry_exact_ties_and_one_ulp_pairs():
    for dim in WIDTHS:
        _, _, (_, vec) = width_catalogue(dim)
        assert (vec[10:20] == vec[0:10]).all()
        d = (vec[20:30] != vec[0:10]).sum(1)
        assert (d == 1).all(), dim


# ---- the "nerualcf" kernels' instantiations ---------------------------------------------------------------------
def _pairs(fname, macro):
    with open(os.path.join(CSRC, fname)) as f:
        return sorted({(int(e), int(h)) for e, h in re.findall(macro + r"\((\d+), (\d+)\)", f.read())})


def test_the_page_dispatches_every_ncf_instantiation_and_the_gpu_cases_reach_them():
    from test_gpu_kernel_matrix import instantiation
    from test_gpu_page_bounds import NCF_PAGE_CASES
    rfy = _pairs("recforyou.cu", "RFY_NCF_CASE")
    assert len(rfy) == 8 and rfy == _pairs("ncf.cu", "SRS_NCF_CASE")
    for model in ("neuralcf", "twotowers"):
        reached = sorted({instantiation(c)[1:] for c in NCF_PAGE_CASES if c.model == model})
        assert reached == rfy, (model, sorted(set(rfy) - set(reached)))


# ---- hand-worked answers on the device tests' catalogues -----------------------------------------------------
def _oracle(movies, ratings, emb=None):
    return recall_oracle(movies, ratings, emb)


@pytest.mark.parametrize("kind", [1, 32, 33, 256, 257])
def test_genre_catalogue_candidate_counts(kind):
    movies, ratings, _, q, max_cands = genre_catalogue(kind)
    c = _oracle(movies, ratings)
    lists = [sum(min(len(c.index[g]), S.GENRE_TOP) for g in gl) for gl in c.genres]
    assert max(lists) == max_cands == lists[0]
    want = {1: 0, 32: 31, 33: 32, 256: 253, 257: 254}[kind]    # the lists less movie 0 in each
    assert len(c.candidates(0)) == want
    if kind in (256, 257):             # genres of exactly 99 / 100 / 101 movies
        assert sorted(len(c.index[g]) for g in "ABC") == ([57, 99, 100] if kind == 256 else [57, 100, 101])
    assert c.rec_list(int(q[-2]), 10, "default")[0] == []        # the genreless movie


def test_the_64_genre_catalogue():
    movies, ratings, _, q, _ = genre_catalogue(6400)
    c = _oracle(movies, ratings)
    assert len(c.index) == 64 and min(len(v) for v in c.index.values()) >= 101
    assert all(c.movies_by_genre(g)[0] == 0 for g in c.index)      # the all-genre movie leads every list
    assert len(c.candidates(0)) == 64 * 99                         # 64 lists of 100, itself in each
    assert len(c.candidates(1)) == 100 and len(c.candidates(2)) == 199 and len(c.candidates(3)) == 199
    # movie 0 heads both lists of movie 3 (G40, G63): only a genre mask wider than 32 bits keeps its second copy out
    assert all(c.movies_by_genre(g, R.MULTI_GENRE_TOP)[0] == 0 for g in ("G40", "G63"))
    assert max(sum(min(len(c.index[g]), 100) for g in gl) for gl in c.genres) == 6400
    # MULTIPLE: 64 lists of 20 and the two global lists of 100 - 1 480 entries, np 2 048
    assert sum(min(len(c.index[g]), R.MULTI_GENRE_TOP) for g in c.genres[0]) + 2 * R.GLOBAL_TOP == 1480


@pytest.mark.parametrize("n", [1, 31, 32, 1023, 1024, 1025, 10_001])
def test_recall_pool_cut(n):
    movies, ratings, emb = flat_catalogue(n)
    c = _oracle(movies, ratings, emb)
    pool = c.get_movies(R.POOL, "rating")
    assert len(pool) == min(n, R.POOL)
    if n > R.POOL:                     # a tie across the cut
        assert c.avg[pool[-1]] == c.avg[c.get_movies(R.POOL + 1, "rating")[-1]]
    ids, _, st = c.embedding_recall(int(movies["movieId"][0]), R.POOL + 1)
    assert st == S.OK and len(ids) == len(pool)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 512, 513, 800])
def test_recforyou_candidates_at_each_sort_width(n):
    movies, ratings, emb = flat_catalogue(n)
    page = RF.RecForYou(_oracle(movies, ratings, emb), [1, 2], [1], [emb[1][0]], cosine=S.warp_cosine_many)
    assert len(page.candidates()) == min(n, RF.CANDIDATES)
    ids, scores, st = page.rec_list(1, 1000, "default")
    assert st == RF.OK and scores == [float(n - i) for i in range(n)]


def test_small_multi_catalogue_puts_every_movie_in_both_global_lists():
    movies, ratings, emb = small_multi_catalogue()
    c = _oracle(movies, ratings, emb)
    assert sorted(c.get_movies(100, "rating")) == sorted(c.get_movies(100, "releaseYear")) == list(range(40))
    ids, scores, _ = c.rec_list(int(movies["movieId"][0]), 100, "default", "multiple")
    nan = [i for i, s in zip(ids, scores) if s != s]
    assert len(ids) == 39 and len(nan) == 9 and ids[:9] == sorted(nan)


@pytest.mark.parametrize("T, want", [(3, [0, 1, 2, -1, -1]), (9, [0, 1, 2, 3, 4]), (10, [0, 2, 3, 4, 5]),
                                     (50, [0, 11, 22, 33, 44])])
def test_history_positions(T, want):
    keys = history_keys(T)
    for model in ("din", "dien"):
        spec = default_spec(model, hist_len=T)
        assert history_positions(spec) == want
        assert [keys.index("userRatedMovie%d" % k) if "userRatedMovie%d" % k in keys else -1
                for k in range(1, 6)] == want
        assert read_history_keys(spec) == ["userRatedMovie%d" % (k + 1) for k in range(5) if want[k] >= 0]
    assert history_positions(default_spec("widendeep")) == [0, -1, -1, -1, -1]
    assert history_positions(default_spec("deepfm")) == [-1] * 5
