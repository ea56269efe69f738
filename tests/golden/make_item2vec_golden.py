"""Regenerate the item2vec fixtures from the reference checkout and check the pins DESIGN.md section 4.12 states.

Run on a machine that has the reference (the GPU machines do not):

    python tests/golden/make_item2vec_golden.py              # a few minutes: four full runs of the C oracle

Checks, on the whole of the reference's ratings.csv:

* the corpus facts (ratings, users, positives, the longest sentence, users with 9- and 10-digit timestamps);
* vocabulary: minCount 5 over the positive ratings keeps exactly the ids of the shipped item2vecEmb.csv;
* user embeddings: every row of the shipped userEmb.csv is the float32 sum of the shipped item vectors over all
  the user's ratings, in reverse file order, with no division;
* text: `embedding.write_embeddings_csv` re-emits both shipped files byte for byte.

Writes, next to this file:

* `item2vec_corpus.npz` - the 657 069 positive movies in sentence order and, per user with a positive rating
  (ascending), the user id and the sentence length, packed so that they compress well (`encode_corpus`; the tests
  read them with `test_item2vec_oracle.corpus`): `ids` (uint16) the distinct movies by count descending, ties by
  id; the movie at each position is `ids[rank_hi * 256 + rank_lo]` (two uint8 planes); `user_step` (uint16) each
  user id minus the previous one (the first minus 0); `length` (uint16) each user's positive ratings.
* `item2vec_user_emb.npz` - the shipped userEmb.csv rows of the users of `featureeng_ratings.npz`: `user` (int32)
  and `line` (the raw text lines).
* `item2vec_fit.json` - for C-oracle seeds 0..3 at the script's configuration (vector size 10, window 5, 10
  iterations, one partition) on the corpus: each seed's mean top-10 cosine-neighbour overlap with every other seed
  and with the shipped vectors, the median vector norm, and the oracle's wall time.
"""
import csv
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

REF = "/root/reference/src/main/resources/webroot/"
SEEDS = (0, 1, 2, 3)


def all_ratings():
    with open(REF + "sampledata/ratings.csv", newline="") as f:
        rows = list(csv.reader(f))[1:]
    u, m, r, t = zip(*rows)
    half = np.array([float(x) * 2 for x in r])
    assert np.array_equal(half, np.rint(half))
    return {"userId": np.array(u, np.int64), "movieId": np.array(m, np.int64), "half": half.astype(np.int64),
            "timestamp": np.array(t, np.int64), "ts_text": t}


def top10(vec):
    """Each row's 10 nearest rows by cosine similarity, itself excluded."""
    x = vec.astype(np.float64)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    s = x @ x.T
    np.fill_diagonal(s, -np.inf)
    return np.argsort(-s, axis=1, kind="stable")[:, :10]


def overlap(a, b):
    return float(np.mean([len(set(x) & set(y)) / 10.0 for x, y in zip(a.tolist(), b.tolist())]))


def encode_corpus(movie, users, lengths):
    """The layout of item2vec_corpus.npz (module docstring)."""
    ids, inv = np.unique(movie, return_inverse=True)
    cnt = np.bincount(inv)
    order = np.lexsort((ids, -cnt))
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    r = rank[inv]
    assert len(ids) <= 65536 and ids.max() < 65536 and np.diff(np.r_[0, users]).max() < 65536 \
        and lengths.max() < 65536
    return {"ids": ids[order].astype(np.uint16), "rank_hi": (r >> 8).astype(np.uint8),
            "rank_lo": (r & 255).astype(np.uint8), "user_step": np.diff(np.r_[0, users]).astype(np.uint16),
            "length": np.asarray(lengths).astype(np.uint16)}


def main():
    from oracle import item2vec as I
    from oracle import item2vec_cext as X
    from sparrowrecsys_b200.embedding import write_embeddings_csv
    from sparrowrecsys_b200.ranking import load_embeddings_csv
    r = all_ratings()
    user, movie, half, ts = r["userId"], r["movieId"], r["half"], r["timestamp"]
    pos = half >= 7
    per_user = np.bincount(user[pos])
    digits = np.array([len(t) for t in r["ts_text"]])
    both = np.intersect1d(np.unique(user[pos & (digits == 9)]), np.unique(user[pos & (digits == 10)]))
    facts = {"ratings": len(user), "users": len(np.unique(user)), "positives": int(pos.sum()),
             "positive_users": int((per_user > 0).sum()), "longest_sentence": int(per_user.max()),
             "users_with_9_and_10_digit_timestamps": len(both)}
    print(facts)
    assert facts == {"ratings": 1168638, "users": 29776, "positives": 657069, "positive_users": 29375,
                     "longest_sentence": 302, "users_with_9_and_10_digit_timestamps": 704}

    users, seqs = I.positive_sequences(user, movie, half, ts)
    ids, counts = I.build_vocab(seqs)
    item_path, user_path = REF + "modeldata/item2vecEmb.csv", REF + "modeldata/userEmb.csv"
    sid, svec = load_embeddings_csv(item_path)
    assert len(ids) == 881 and set(ids.tolist()) == set(sid.tolist()), "vocabulary pin"
    code, point, codelen = I.huffman(counts)
    print("vocabulary pin: %d ids; trainWordsCount %d; deepest Huffman code %d"
          % (len(ids), counts.sum(), codelen.max()))

    uid, uvec = load_embeddings_csv(user_path)
    ou, ovec = I.user_embeddings(user, movie, sid, svec)
    order = np.argsort(uid)
    assert np.array_equal(ou, uid[order]) and np.array_equal(ovec.view(np.int32), uvec[order].view(np.int32)), \
        "user-embedding pin"
    print("user-embedding pin: all %d rows bit for bit" % len(uid))

    for path, (i, v) in ((item_path, (sid, svec)), (user_path, (uid, uvec))):
        out = os.path.join("/tmp", "item2vec_golden_%d.csv" % os.getpid())
        write_embeddings_csv(out, i, v)
        with open(out) as f, open(path) as g:
            assert f.read() == g.read(), "text pin: " + path
        os.remove(out)
    print("text pin: %d values re-emitted byte for byte" % (svec.size + uvec.size))

    from test_item2vec_oracle import corpus as read_corpus
    corpus = encode_corpus(np.concatenate(seqs), users, np.array([len(s) for s in seqs]))
    np.savez_compressed(os.path.join(HERE, "item2vec_corpus.npz"), **corpus)
    back = read_corpus()
    assert np.array_equal(back[0], np.concatenate(seqs)) and np.array_equal(back[1], users)
    assert np.array_equal(np.diff(back[2]), [len(s) for s in seqs])
    fixture_users = np.unique(np.load(os.path.join(HERE, "featureeng_ratings.npz"))["userId"]).astype(np.int64)
    with open(user_path) as f:
        lines = f.readlines()
    keep = [ln for ln in lines if int(ln.split(":")[0]) in set(fixture_users.tolist())]
    keep.sort(key=lambda ln: int(ln.split(":")[0]))
    np.savez_compressed(os.path.join(HERE, "item2vec_user_emb.npz"),
                        user=np.array([int(ln.split(":")[0]) for ln in keep], np.int32), line=np.array(keep))
    print("fixtures: corpus %d words (%d bytes), %d user rows"
          % (len(back[0]), os.path.getsize(os.path.join(HERE, "item2vec_corpus.npz")), len(keep)))

    words, woffs = I.chunk_corpus(seqs, ids)
    runs, secs = {}, {}
    for seed in SEEDS:
        t0 = time.perf_counter()
        runs[seed] = X.train(words, woffs, counts, code, point, codelen, 10, 5, 10, 1, seed)
        secs[seed] = time.perf_counter() - t0
        print("seed %d: %.1f s" % (seed, secs[seed]))
    where = {m: i for i, m in enumerate(ids.tolist())}
    shipped = top10(svec[np.argsort([where[m] for m in sid.tolist()])])
    nb = {s: top10(v) for s, v in runs.items()}
    fit = {"configuration": {"vector_size": 10, "window": 5, "iterations": 10, "partitions": 1},
           "words": int(len(words)), "vocabulary": int(len(ids)),
           "shipped_median_norm": float(np.median(np.linalg.norm(svec, axis=1))), "seeds": {}}
    for s in SEEDS:
        fit["seeds"][str(s)] = {
            "overlap_with_seeds": {str(o): overlap(nb[s], nb[o]) for o in SEEDS if o != s},
            "overlap_with_shipped": overlap(nb[s], shipped),
            "median_norm": float(np.median(np.linalg.norm(runs[s], axis=1))),
            "oracle_seconds": round(secs[s], 2)}
    print(json.dumps(fit, indent=1))
    with open(os.path.join(HERE, "item2vec_fit.json"), "w") as f:
        json.dump(fit, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
