"""The sample builder's numpy oracle (oracle/feature_eng.py) against the reference's own output.

`featureeng_model_samples.npz` holds the rows of modelSamples.csv, a 10 % sample of FeatureEngForRecModel's rows,
for the users whose ratings `featureeng_ratings.npz` holds (the 5 000 smallest user ids of ratings.csv; a user's
window depends on that user's ratings only).  The movie features span every user, so they are checked on their
own, from each movie's rating moments over the whole of ratings.csv (`featureeng_movies.npz`).  Spark orders a
user's equal timestamps by its shuffles, so rows are classed by the ties around them (`tie_classes`):

* tie-free: no two ratings of the user share a timestamp among the window's rows, the row itself, the row after it
  and the row before the window - the window's contents and order are then unique, and every column must match;
* interior ties: the ties lie strictly inside the window - its contents are unique, so the order-free columns must
  match, and the history / genre lists up to a permutation within tied positions;
* edge ties: the row's own position or the window's edge is tied - only the row's own columns are defined.
"""
import os

import numpy as np
import pytest

from oracle import feature_eng as F
from sparrowrecsys_b200 import featureeng as FE
from sparrowrecsys_b200.features import genre_to_index

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MOVIE_STAT_COLS = ("movieRatingCount", "movieAvgRating", "movieRatingStddev")      # over all users' ratings
ROW_COLS = ("movieId", "userId", "rating", "timestamp", "label", "releaseYear", "movieGenre1", "movieGenre2",
            "movieGenre3")
WINDOW_FREE_COLS = ("userRatingCount", "userAvgReleaseYear", "userReleaseYearStddev", "userAvgRating",
                    "userRatingStddev")
TIE_FREE, INTERIOR, EDGE = 0, 1, 2


def fixture_inputs():
    r = np.load(os.path.join(GOLDEN, "featureeng_ratings.npz"))
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    ratings = {"userId": r["userId"].astype(np.int32), "movieId": r["movieId"].astype(np.int32),
               "rating": r["half"] / 2.0, "timestamp": r["timestamp"].astype(np.int32)}
    movies = {"movieId": m["movieId"], "title": m["title"].tolist(), "genres": m["genres"].tolist()}
    return ratings, movies


def model_samples():
    z = np.load(os.path.join(GOLDEN, "featureeng_model_samples.npz"))
    return ({k: (z[k].astype(object) if z[k].dtype.kind == "U" else z[k]) for k in F.COLUMNS}, z["text"])


def all_movie_features():
    """movie id -> (movieRatingCount, movieAvgRating, movieRatingStddev) over the whole of ratings.csv."""
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    avg_k, std_k = F.movie_features(m["all_count"], m["all_sum_half"], m["all_sum_half2"])
    return m["all_count"].astype(np.int32), F.hundredths_to_f32(avg_k), F.hundredths_to_f32(std_k)


def sorted_order(ratings):
    ts = np.asarray(ratings["timestamp"], np.int64)
    digits = np.array([len(str(t)) for t in ts.tolist()])
    return np.lexsort((np.arange(len(ts)), digits, ts * 10 ** (10 - digits), np.asarray(ratings["userId"])))


def tie_classes(ratings):
    """Per ratings row (file order): TIE_FREE, INTERIOR or EDGE, and the window start in sorted order."""
    order = sorted_order(ratings)
    N = len(order)
    su, st = np.asarray(ratings["userId"])[order], np.asarray(ratings["timestamp"])[order]
    start = np.flatnonzero(np.r_[True, su[1:] != su[:-1]])
    seg = np.repeat(start, np.diff(np.r_[start, N]))
    i = np.arange(N)
    lo = np.maximum(seg, i - F.WINDOW)
    pair = np.r_[False, (su[1:] == su[:-1]) & (st[1:] == st[:-1])]        # pair[p]: rows p - 1 and p tie
    P = np.r_[0, np.cumsum(pair)]
    count = lambda a, b: P[np.clip(b, 0, N)] - P[np.clip(a, 0, N)]       # pairs p in [a, b)
    any_tie = count(lo, i + 2) > 0                                        # pairs lo .. i + 1
    interior = count(lo + 1, i) == count(lo, i + 2)                       # all of them inside (lo, i - 1]
    cls = np.where(~any_tie, TIE_FREE, np.where(interior, INTERIOR, EDGE))
    back = np.empty(N, np.int64)
    back[order] = i
    return cls[back], order, lo, back


@pytest.fixture(scope="module")
def full():
    ratings, movies = fixture_inputs()
    out = F.build_samples(ratings, movies)
    ms, _ = model_samples()
    cls, order, lo, back = tie_classes(ratings)
    key = lambda u, m: np.asarray(u, np.int64) * 100000 + np.asarray(m, np.int64)   # a user rates a movie once
    kf = key(ratings["userId"], ratings["movieId"])
    assert len(np.unique(kf)) == len(kf)
    sf = np.argsort(kf)
    file_row = sf[np.searchsorted(kf[sf], key(ms["userId"], ms["movieId"]))]
    assert np.array_equal(kf[file_row], key(ms["userId"], ms["movieId"]))
    ko = key(out["userId"], out["movieId"])
    so = np.argsort(ko)
    pos = np.searchsorted(ko[so], key(ms["userId"], ms["movieId"]))
    pos = np.minimum(pos, len(ko) - 1)
    out_row = np.where(ko[so[pos]] == key(ms["userId"], ms["movieId"]), so[pos], -1)
    return dict(ratings=ratings, movies=movies, out=out, ms=ms, cls=cls[file_row], out_row=out_row,
                order=order, lo=lo, back=back, file_row=file_row)


def test_tie_class_counts(full):
    """The counts DESIGN.md section 4.11 records."""
    cls = full["cls"]
    assert len(cls) == 19381
    assert [(cls == c).sum() for c in (TIE_FREE, INTERIOR, EDGE)] == [6858, 4140, 8383]


def test_every_column_of_every_tie_free_row(full):
    sel = np.flatnonzero(full["cls"] == TIE_FREE)
    assert (full["out_row"][sel] >= 0).all()
    rows = full["out_row"][sel]
    for c in F.COLUMNS:
        if c in MOVIE_STAT_COLS:
            continue
        a, b = full["out"][c][rows], full["ms"][c][sel]
        assert a.dtype == b.dtype or (a.dtype == object and b.dtype == object), c
        assert np.array_equal(a, b), (c, np.flatnonzero(a != b)[:5])


def test_movie_features_of_every_model_samples_movie():
    """The movie columns of all 110 778 modelSamples rows (one feature row per movie) from the movies' moments."""
    z = np.load(os.path.join(GOLDEN, "featureeng_model_samples.npz"))["movie_columns"]
    m = np.load(os.path.join(GOLDEN, "featureeng_movies.npz"))
    avg_k, std_k = F.movie_features(m["all_count"], m["all_sum_half"], m["all_sum_half2"])
    ids = z[:, 0]
    assert len(ids) > 900
    assert np.array_equal(m["all_count"][ids], z[:, 1])
    assert np.array_equal(avg_k[ids], z[:, 2]) and np.array_equal(std_k[ids], z[:, 3])
    count, avg, std = all_movie_features()
    ms, _ = model_samples()
    mv = ms["movieId"]
    assert np.array_equal(count[mv], ms["movieRatingCount"])
    assert np.array_equal(avg[mv], ms["movieAvgRating"]) and np.array_equal(std[mv], ms["movieRatingStddev"])


def _groups_match(ours, theirs, key_of, pool):
    """`ours` and `theirs` (lists of ids, 0 / "" = none) agree up to permutation within equal keys: the key
    sequences are equal, each complete key group holds the same ids, and the last group (which the list's end may
    cut) holds ids of the pool's group with that key."""
    ko, kt = [key_of(x) for x in ours], [key_of(x) for x in theirs]
    if ko != kt:
        return False
    for k in set(ko):
        a = {x for x, kk in zip(ours, ko) if kk == k}
        b = {x for x, kk in zip(theirs, kt) if kk == k}
        full_group = {x for x in pool if key_of(x) == k}
        if a != b and not (ko[-1] == k and b <= full_group and len(a) == len(b)):
            return False
    return True


def test_interior_tied_rows(full):
    """Order-free columns equal; userRatedMovie and userGenre equal up to permutation within tied positions."""
    sel = np.flatnonzero(full["cls"] == INTERIOR)
    rows = full["out_row"][sel]
    assert (rows >= 0).all()
    out, ms = full["out"], full["ms"]
    for c in ROW_COLS + WINDOW_FREE_COLS:
        assert np.array_equal(out[c][rows], ms[c][sel]), c
    ratings, movies = full["ratings"], full["movies"]
    order, lo, back = full["order"], full["lo"], full["back"]
    glist = {int(m): g.split("|") for m, g in zip(movies["movieId"], movies["genres"])}
    ts = np.asarray(ratings["timestamp"])
    mv = np.asarray(ratings["movieId"])
    pos = np.asarray(ratings["rating"]) >= 3.5
    bad = []
    for s, r in zip(sel.tolist(), rows.tolist()):
        i = back[full["file_row"][s]]
        win = order[lo[i]:i]
        pw = win[pos[win]]
        mts = {int(mv[f]): int(ts[f]) for f in pw}
        rated = lambda d, row: [int(d["userRatedMovie%d" % k][row]) for k in range(1, 6)]
        if not _groups_match(rated(out, r), rated(ms, s), lambda m: mts.get(m), list(mts)):
            bad.append(("rated", s))
        cnt = {}
        for f in pw:
            for g in glist.get(int(mv[f]), []):
                cnt[g] = cnt.get(g, 0) + 1
        genres = lambda d, row: [d["userGenre%d" % k][row] for k in range(1, 6)]
        if not _groups_match(genres(out, r), genres(ms, s), lambda g: cnt.get(g, 0), list(cnt)):
            bad.append(("genre", s))
    assert not bad, bad[:10]


def test_edge_tied_rows_match_their_own_columns(full):
    sel = np.flatnonzero((full["cls"] == EDGE) & (full["out_row"] >= 0))
    rows = full["out_row"][sel]
    for c in ROW_COLS:
        assert np.array_equal(full["out"][c][rows], full["ms"][c][sel]), c


@pytest.mark.parametrize("name", ["neuralcf_trainset", "deepfm_trainset"])
def test_tie_free_rows_of_the_fit_trainsets(full, name):
    """The rows `fit` is tested on (trainingSamples.csv, another sample of the same job) match where tie-free."""
    zz = np.load(os.path.join(GOLDEN, name + ".npz"))
    ratings = full["ratings"]
    mine = np.isin(zz["userId"], ratings["userId"])
    z = {k: zz[k][mine] for k in zz.files}
    movie_stats = dict(zip(MOVIE_STAT_COLS, all_movie_features()))
    cls, order, lo, back = tie_classes(ratings)
    key = lambda u, m: np.asarray(u, np.int64) * 100000 + np.asarray(m, np.int64)
    kf = key(ratings["userId"], ratings["movieId"])
    sf = np.argsort(kf)
    fr = sf[np.searchsorted(kf[sf], key(z["userId"], z["movieId"]))]
    assert np.array_equal(kf[fr], key(z["userId"], z["movieId"]))
    tf = cls[fr] == TIE_FREE
    assert tf.sum() > 2000
    out = full["out"]
    ko = key(out["userId"], out["movieId"])
    so = np.argsort(ko)
    rows = so[np.searchsorted(ko[so], key(z["userId"], z["movieId"])[tf])]
    for c in z:
        a = movie_stats[c][z["movieId"][tf]] if c in MOVIE_STAT_COLS else out[c][rows]
        if c in ("movieGenre1", "userGenre1"):
            a = genre_to_index(a).astype(np.int8)
        assert np.array_equal(a, z[c][tf]), c


# ---- known answers on hand-built inputs (tests/test_gpu_featureeng.py runs them on the device) -------------------
def hand_inputs():
    """Users: 1 mixed 9/10-digit timestamps, 2 one rating, 3 a 103-rating history, 4 all negative, 5 and 6 exact
    HALF_EVEN ties of userAvgRating, 7 short titles, a movie missing from movies.csv and "(no genres listed)"."""
    R = []                                                               # (user, movie, rating, timestamp)
    R += [(1, 1, 4.0, 1000000000), (1, 2, 3.0, 999999999), (1, 3, 5.0, 1000000001)]
    R += [(2, 4, 5.0, 1000000000)]
    R += [(3, 10 + k, 5.0 if k < 3 else 1.0, 1000000001 + k) for k in range(103)]
    R += [(4, 1 + k, 2.0, 1100000000 + k) for k in range(3)]
    R += [(5, 1 + k, 3.0 if k == 7 else 2.0, 1200000000 + k) for k in range(9)]
    R += [(6, 1 + k, 3.0 if 5 <= k < 8 else 2.0, 1200000000 + k) for k in range(9)]
    R += [(7, 200, 4.0, 1300000000), (7, 201, 4.5, 1300000001), (7, 202, 5.0, 1300000002), (7, 203, 1.0, 1300000003)]
    u, m, r, t = zip(*R)
    ratings = {"userId": np.array(u, np.int32), "movieId": np.array(m, np.int32), "rating": np.array(r),
               "timestamp": np.array(t, np.int32)}
    titles = {1: "Toy Story (1995)", 2: "Heat (1995)", 3: "Casino (1995)", 4: "Up", 200: "Alien (1979)",
              201: "Short", 202: "Blade Runner (1982)"}
    genres = {1: "Animation|Comedy", 2: "Action|Crime", 3: "Crime|Drama", 4: "Comedy", 200: "Horror|Sci-Fi",
              201: "(no genres listed)", 202: "Sci-Fi"}
    for k in range(113):
        titles.setdefault(10 + k, "Movie %d (2000)" % k)
        genres.setdefault(10 + k, "Drama")
    ids = sorted(titles)                                                 # movie 203 is missing from movies.csv
    movies = {"movieId": np.array(ids, np.int32), "title": [titles[i] for i in ids],
              "genres": [genres[i] for i in ids]}
    return ratings, movies


HAND_EXPECTED = {                      # (userId, movieId) -> columns of that row; rows not listed are dropped
    (1, 2): {"userRatingCount": 2, "userRatedMovie1": 3, "userRatedMovie2": 1, "userRatedMovie3": 0,
             "userAvgRating": 4.5, "userRatingStddev": 0.71, "userGenre1": "Crime", "userGenre2": "Drama",
             "userGenre3": "Comedy", "userGenre4": "Animation", "userGenre5": ""},
    (3, 112): {"userRatingCount": 100, "userRatedMovie1": 12, "userRatedMovie2": 0, "userAvgRating": 1.04,
               "userAvgReleaseYear": 2000.0, "userReleaseYearStddev": 0.0},
    (3, 111): {"userRatingCount": 100, "userRatedMovie1": 12, "userRatedMovie2": 11, "userRatedMovie3": 0},
    (3, 12): {"userRatingCount": 2, "userRatedMovie1": 11, "userRatedMovie2": 10, "userGenre1": "Drama"},
    (4, 3): {"userRatingCount": 2, "userRatedMovie1": 0, "userRatedMovie5": 0, "userGenre1": "", "label": 0,
             "userRatingStddev": 0.0, "userAvgRating": 2.0},
    (5, 9): {"userRatingCount": 8, "userAvgRating": 2.12},                # 17 / 8 = 2.125 -> HALF_EVEN 2.12
    (6, 9): {"userRatingCount": 8, "userAvgRating": 2.38},                # 19 / 8 = 2.375 -> 2.38
    (7, 202): {"userRatingCount": 2, "userRatedMovie1": 201, "userRatedMovie2": 200,
               "userAvgReleaseYear": 1984.0, "userReleaseYearStddev": 7.78, "releaseYear": 1982,
               "userGenre1": "Sci-Fi", "userGenre2": "Horror", "userGenre3": "(no genres listed)",
               "movieRatingCount": 1, "movieRatingStddev": 0.0, "movieAvgRating": 5.0},
    (7, 203): {"userRatingCount": 3, "userRatedMovie1": 202, "releaseYear": 1990, "movieGenre1": "",
               "userGenre1": "Sci-Fi", "userGenre2": "Horror", "userGenre3": "(no genres listed)", "label": 0},
}


def check_hand(out):
    """The rows `out` holds are exactly HAND_EXPECTED's keys plus the other kept rows, with the listed values."""
    got = {(int(u), int(m)): r for r, (u, m) in enumerate(zip(out["userId"], out["movieId"]))}
    for key, cols in HAND_EXPECTED.items():
        assert key in got, key
        for c, v in cols.items():
            x = out[c][got[key]]
            if isinstance(v, float):
                assert x == np.float32(float("%.2f" % v)), (key, c, x, v)
            else:
                assert x == v, (key, c, x, v)
    assert not any(k[0] == 2 for k in got)                               # one rating: filtered
    assert (1, 1) not in got and (1, 3) not in got                       # "999999999" sorts after "1000000001"
    assert len(got) == 1 + 101 + 1 + 7 + 7 + 2                           # kept rows of users 1, 3, 4, 5, 6, 7


def test_hand_built_known_answers():
    ratings, movies = hand_inputs()
    out = F.build_samples(ratings, movies)
    check_hand(out)
    assert set(out) == set(F.COLUMNS)


# ---- the rules one by one ----------------------------------------------------------------------------------------
def test_title_rule():
    for title, year in (("Toy Story (1995)", 1995), ("Up", 1990), ("(1995)", 1995), ("Short", 1990),
                        (None, 1990), ("  abc  ", 1990), ("Seven (a.k.a. Se7en) (1995)", 1995)):
        assert F.release_year(title) == year == FE.release_year(title), title
    for title in ("Heat (1995) ", " (1995)", "Shorty", "No year here"):   # the reference's substring / toInt throw
        with pytest.raises(ValueError):
            F.release_year(title)
        with pytest.raises(ValueError):
            FE.release_year(title)


def test_format_number_half_even_on_the_binary_value():
    x = np.array([2.125, 2.375, 0.125, 0.285, 1.005, 2.675, 0.5, 0.0, 999.995, 3.14159])
    assert F.format2_hundredths(x).tolist() == [212, 238, 12, 28, 100, 267, 50, 0, 100000, 314]
    assert F.format2_text(1234.5) == "1,234.50" and F.format2_text(3.5) == "3.50"


def test_hundredths_to_float32_is_what_the_csv_text_parses_to():
    k = np.arange(0, 100000)
    text = np.array(["%d.%02d" % (a // 100, a % 100) for a in k.tolist()])
    assert np.array_equal(F.hundredths_to_f32(k), text.astype(np.float64).astype(np.float32))


def test_hashmap_closed_form_matches_the_table():
    rng = np.random.default_rng(7)
    words = ["Adventure", "Animation", "Children", "Comedy", "Fantasy", "Romance", "Drama", "Action", "Crime",
             "Thriller", "Horror", "Mystery", "Sci-Fi", "IMAX", "Documentary", "War", "Musical", "Western",
             "Film-Noir", "(no genres listed)"]
    h = [F.java_string_hash(w) for w in words]
    assert F.java_string_hash("Drama") == 66292295 and FE.java_string_hash("Drama") == 66292295
    b16, b32 = F.genre_buckets(h)
    for _ in range(400):
        n = int(rng.integers(1, len(words) + 1))
        seq = [int(x) for x in rng.permutation(len(words))[:n]]
        want = F.scala_hashmap_keys([words[i] for i in seq])
        ins = np.empty(len(words), np.int64)
        ins[seq] = np.arange(n)
        keys = F._genre_order_keys(ins[seq], n, b16[seq], b32[seq])
        got = [words[seq[j]] for j in np.argsort(keys, kind="stable")]
        assert got == want, (seq, got, want)


def test_write_samples_csv_reproduces_model_samples_text(tmp_path):
    ms, text = model_samples()
    n = len(text) - 1
    path = tmp_path / "s.csv"
    FE.write_samples_csv(str(path), {k: v[:n] for k, v in ms.items()})
    assert path.read_text().splitlines(keepends=True) == [t.replace("\r\n", "\n") for t in text.tolist()]


def test_build_samples_rejects_before_the_device():
    ratings, movies = hand_inputs()
    bad = dict(ratings, rating=ratings["rating"] + 0.25)
    with pytest.raises(ValueError):
        FE.build_samples(bad, movies)
    bad = dict(ratings, movieId=-ratings["movieId"])
    with pytest.raises(ValueError):
        FE.build_samples(bad, movies)
