"""Regenerate the sample-builder fixtures from the reference checkout.

Run on a machine that has the reference (the GPU machines do not):

    python tests/golden/make_featureeng_golden.py            # about half a minute

The reference's ratings.csv (1 168 638 ratings of 29 776 users) is too large to keep whole, so the fixtures hold
the users with the USERS smallest ids - a user's window features depend on that user's ratings only - and, for
the movie features, which span every user, each movie's rating moments over the whole file.  Writes, next to this
file:

* `featureeng_ratings.npz` - every rating of those users, in ratings.csv order: `userId`, `movieId` (uint16),
  `half` (uint8, the rating in half-stars) and `timestamp` (uint32).
* `featureeng_movies.npz` - movies.csv: `movieId` (int32), `title` and `genres` (unicode); and, over all of
  ratings.csv, per movie id m in 0..max: `all_count`, `all_sum_half`, `all_sum_half2` (int64: count, sum of
  half-stars, sum of their squares).
* `featureeng_model_samples.npz` - the rows of modelSamples.csv (a 10 % sample of FeatureEngForRecModel's output)
  of those users: the 27 columns as `features.load_samples_csv` reads them (genre columns as unicode) and `text`,
  the raw lines of the first TEXT_ROWS of them (header first); and, from all 110 778 rows, `movie_columns`
  [movies][4] = movieId, movieRatingCount and the two-decimal movie columns times 100 (one row per movie).

It also prints the tie classes (tests/test_featureeng_oracle.py) of all 110 778 modelSamples rows, which DESIGN.md
section 4.11 records, and checks that the oracle run on the whole of ratings.csv matches every column of every
tie-free one.  `--check` rebuilds the three files and compares them with the committed ones.
"""
import csv
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

REF = "/root/reference/src/main/resources/webroot/sampledata/"
USERS = 5000
TEXT_ROWS = 2000


def all_ratings():
    with open(REF + "ratings.csv", newline="") as f:
        rows = list(csv.reader(f))[1:]
    u, m, r, t = (np.array(c) for c in zip(*rows))
    half = np.array([float(x) * 2 for x in r])
    assert np.array_equal(half, np.rint(half))
    return {"userId": u.astype(np.uint16), "movieId": m.astype(np.uint16), "half": half.astype(np.uint8),
            "timestamp": t.astype(np.int64).astype(np.uint32)}


def kept_users(r):
    return np.unique(r["userId"])[:USERS]


def movies(r):
    with open(REF + "movies.csv", newline="", encoding="utf-8") as f:
        rows = list(csv.reader(f))[1:]
    m, h = r["movieId"].astype(np.int64), r["half"].astype(np.int64)
    return {"movieId": np.array([int(x[0]) for x in rows], np.int32),
            "title": np.array([x[1] for x in rows]), "genres": np.array([x[2] for x in rows]),
            "all_count": np.bincount(m), "all_sum_half": np.bincount(m, weights=h).astype(np.int64),
            "all_sum_half2": np.bincount(m, weights=h * h).astype(np.int64)}


def model_samples(users):
    from sparrowrecsys_b200 import features
    s = features.load_samples_csv(REF + "modelSamples.csv")
    keep = np.isin(s["userId"], users)
    out = {k: (v.astype(str) if v.dtype == object else v)[keep] for k, v in s.items()}
    with open(REF + "modelSamples.csv", newline="") as f:
        lines = f.readlines()
    out["text"] = np.array([lines[0]] + [lines[1 + i] for i in np.flatnonzero(keep)[:TEXT_ROWS].tolist()])
    mc = np.stack([s["movieId"], s["movieRatingCount"], np.rint(s["movieAvgRating"].astype(np.float64) * 100),
                   np.rint(s["movieRatingStddev"].astype(np.float64) * 100)], axis=1).astype(np.int64)
    mc = np.unique(mc, axis=0)
    assert len(np.unique(mc[:, 0])) == len(mc), "a movie with two different feature rows"
    out["movie_columns"] = mc
    return out, s


def check_whole_file(r, s):
    from test_featureeng_oracle import EDGE, INTERIOR, TIE_FREE, tie_classes
    ratings = {"userId": r["userId"].astype(np.int32), "movieId": r["movieId"].astype(np.int32),
               "rating": r["half"] / 2.0, "timestamp": r["timestamp"].astype(np.int32)}
    cls = tie_classes(ratings)[0]
    key = lambda u, m: np.asarray(u, np.int64) * 100000 + np.asarray(m, np.int64)
    kf = key(ratings["userId"], ratings["movieId"])
    sf = np.argsort(kf)
    c = cls[sf[np.searchsorted(kf[sf], key(s["userId"], s["movieId"]))]]
    print("modelSamples rows: tie-free %d, interior ties %d, edge ties %d"
          % tuple((c == k).sum() for k in (TIE_FREE, INTERIOR, EDGE)))
    # the oracle on the whole file against every tie-free row (the tests see the fixture's users only)
    from oracle import feature_eng as F
    m = movies(r)
    out = F.build_samples(ratings, {"movieId": m["movieId"], "title": m["title"].tolist(),
                                    "genres": m["genres"].tolist()})
    ko = key(out["userId"], out["movieId"])
    so = np.argsort(ko)
    tf = np.flatnonzero(c == TIE_FREE)
    rows = so[np.searchsorted(ko[so], key(s["userId"], s["movieId"])[tf])]
    assert np.array_equal(ko[rows], key(s["userId"], s["movieId"])[tf])
    bad = {col: int((out[col][rows] != s[col][tf]).sum()) for col in F.COLUMNS}
    assert not any(bad.values()), bad
    print("the oracle on all of ratings.csv matches every column of all %d tie-free rows" % len(tf))


def main():
    r = all_ratings()
    users = kept_users(r)
    sub = {k: v[np.isin(r["userId"], users)] for k, v in r.items()}
    ms, full_ms = model_samples(users)
    sets = {"featureeng_ratings.npz": sub, "featureeng_movies.npz": movies(r), "featureeng_model_samples.npz": ms}
    for name, d in sets.items():
        path = os.path.join(HERE, name)
        if "--check" in sys.argv:
            old = np.load(path)
            assert sorted(old.files) == sorted(d) and all(np.array_equal(old[k], d[k]) for k in d), name
            print(name, "matches")
        else:
            np.savez_compressed(path, **d)
            print(name, os.path.getsize(path), "bytes")
    check_whole_file(r, full_ms)


if __name__ == "__main__":
    main()
