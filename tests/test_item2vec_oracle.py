"""item2vec's oracles (oracle/item2vec.py, oracle/item2vec_c.c) against the reference's shipped files and known answers.

`item2vec_corpus.npz` holds the 657 069 positive ratings of the reference's ratings.csv in sentence order; fed to the
library as ratings (`corpus_ratings`) it rebuilds that corpus.  `item2vec_user_emb.npz` holds the shipped userEmb.csv
rows of the 5 000 users of `featureeng_ratings.npz`, whose ratings are complete, so those rows depend on fixture data
only.  DESIGN.md section 4.12 gives the semantics.
"""
import ctypes as C
import heapq
import math
import os

import numpy as np
import pytest

from oracle import item2vec as I
from oracle import item2vec_cext as X
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200.embedding import write_embeddings_csv
from sparrowrecsys_b200.ranking import load_embeddings_csv

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAX_RATINGS = 21000000            # the library's bound on n_ratings


def corpus():
    """(movies int64 [N] in sentence order, users int32 [S] ascending, offsets int64 [S + 1]), unpacked from the
    layout tests/golden/make_item2vec_golden.py writes."""
    z = np.load(os.path.join(GOLDEN, "item2vec_corpus.npz"))
    rank = z["rank_hi"].astype(np.int64) * 256 + z["rank_lo"]
    movie = z["ids"].astype(np.int64)[rank]
    user = np.cumsum(z["user_step"].astype(np.int64)).astype(np.int32)
    return movie, user, np.r_[0, np.cumsum(z["length"].astype(np.int64))]


def corpus_ratings(users=None):
    """The corpus as ratings: every rating positive (4.0), timestamp 1 000 000 000 + position, so that string order
    is position order.  `users`: keep the first that many users."""
    movie, user, off = corpus()
    if users is not None:
        off = off[:users + 1]
        user = user[:users]
        movie = movie[:off[-1]]
    n = len(movie)
    return {"userId": np.repeat(user, np.diff(off)).astype(np.int32), "movieId": movie.astype(np.int32),
            "rating": np.full(n, 4.0), "timestamp": (1000000000 + np.arange(n)).astype(np.int32)}


def fixture_ratings():
    r = np.load(os.path.join(GOLDEN, "featureeng_ratings.npz"))
    return {"userId": r["userId"].astype(np.int32), "movieId": r["movieId"].astype(np.int32),
            "rating": r["half"] / 2.0, "timestamp": r["timestamp"].astype(np.int32)}


def halves(r):
    return np.rint(np.asarray(r["rating"]) * 2).astype(np.int64)


def shipped_items():
    return load_embeddings_csv(os.path.join(GOLDEN, "item2vecEmb.csv"))


def shipped_user_rows():
    z = np.load(os.path.join(GOLDEN, "item2vec_user_emb.npz"))
    lines = z["line"].tolist()
    rows = np.array([[float(v) for v in ln.split(":")[1].split()] for ln in lines], np.float32)
    return z["user"], rows, lines


def oracle_c(r, **kw):
    return X.item2vec(r["userId"], r["movieId"], halves(r), r["timestamp"], **kw)


@pytest.fixture(scope="module")
def vocab():
    r = corpus_ratings()
    _, seqs = I.positive_sequences(r["userId"], r["movieId"], halves(r), r["timestamp"])
    ids, counts = I.build_vocab(seqs)
    return seqs, ids, counts


def test_corpus_rebuilds_the_sentences(vocab):
    seqs, _, _ = vocab
    movie, user, off = corpus()
    assert len(seqs) == len(user) == 29375 and len(movie) == 657069
    assert all(np.array_equal(s, movie[a:b]) for s, a, b in zip(seqs, off[:-1], off[1:]))


def test_vocabulary_is_the_shipped_ids(vocab):
    _, ids, counts = vocab
    sid, _ = shipped_items()
    assert len(ids) == 881 and set(ids.tolist()) == set(sid.tolist())
    assert counts.min() >= 5 and np.all(np.diff(counts) <= 0)
    tie = np.diff(counts) == 0
    assert np.all(np.diff(ids)[tie] > 0)                       # ties: movie id ascending


def _optimal_cost(counts):
    h = [int(c) for c in counts]
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        a, b = heapq.heappop(h), heapq.heappop(h)
        cost += a + b
        heapq.heappush(h, a + b)
    return cost


def test_huffman_codes_prefix_free_root_and_optimal(vocab):
    _, ids, counts = vocab
    code, point, codelen = I.huffman(counts)
    V = len(counts)
    words = ["".join(str(int(b)) for b in code[w, :codelen[w]]) for w in range(V)]
    assert len(set(words)) == V
    srt = sorted(words)
    assert not any(b.startswith(a) for a, b in zip(srt, srt[1:]))
    assert np.all(point[:, 0] == V - 2)
    assert np.all((point[:, :codelen.max()] >= 0) | (np.arange(codelen.max())[None, :] >= codelen[:, None]))
    assert int(np.sum(counts * codelen)) == _optimal_cost(counts)
    for w in range(V):                                          # distinct nodes on each path
        assert len(set(point[w, :codelen[w]].tolist())) == codelen[w]
    assert codelen.max() <= 32


def _deepest_counts(depth):
    """The smallest counts (each >= 5) whose tree has a code of `depth`: a caterpillar where every new leaf
    equals the subtree built so far (ties go to the internal node)."""
    c = [5, 5]
    while len(c) < depth + 1:
        c.append(sum(c[:-1]))
    return sorted(c, reverse=True)


def test_a_33_deep_code_needs_more_ratings_than_the_library_takes():
    for depth in (5, 32, 33):
        counts = np.array(_deepest_counts(depth), np.int64)
        _, _, codelen = I.huffman(counts)
        assert codelen.max() == depth
        smaller = counts.copy()
        smaller[0] -= 1                                         # the largest count one less: the tree is shallower
        assert I.huffman(smaller)[2].max() < depth or smaller[0] < 5
    total = int(np.sum(_deepest_counts(33)))
    assert total > MAX_RATINGS, total


def test_exp_table_and_index_edges():
    e = I.exp_table()
    assert e.dtype == np.float32 and e.shape == (1000,)
    t0 = math.exp(-6.0)
    assert e[0] == np.float32(t0 / (t0 + 1))
    assert e[500] == np.float32(0.5)
    assert e[999] == np.float32(math.exp(5.988) / (math.exp(5.988) + 1))
    assert np.all(np.diff(e) >= 0)
    assert I.exp_index(np.nextafter(np.float32(-6), np.float32(0))) == 0
    assert I.exp_index(np.nextafter(np.float32(6), np.float32(0))) == 996      # the float sum rounds to 12.0
    assert I.exp_index(0.0) == 498                                              # 6 * 83, not 500


def test_hand_computed_two_word_vocabulary_single_window():
    """Sentence [w0, w1], window 1, one iteration, counts 1 and 1: the root is node 0, w0's code is 1 and w1's
    is 0.  Pair 1 (centre w0, context w1): f = 0, so g1 = (0 - e[498]) alpha and syn1 = g1 syn0[1].  Pair 2 (centre
    w1, context w0): f = syn0[0].syn1, g2 = (1 - e[ind]) alpha, syn0[0] += g2 syn1."""
    code, point, codelen = I.huffman(np.array([1, 1]))
    assert codelen.tolist() == [1, 1] and code[:, 0].tolist() == [1, 0] and point[:, 0].tolist() == [0, 0]
    D, seed = 4, 11
    s0 = I.init_syn0(seed, 2, D).astype(np.float64)
    e = I.exp_table().astype(np.float64)
    a = 0.025
    g1 = (0 - e[498]) * a
    syn1 = g1 * s0[1]
    f = float(s0[0] @ syn1)
    g2 = (1 - e[int((f + 6) * 83)]) * a
    want0 = s0[0] + g2 * syn1
    got = I.train(np.array([0, 1], np.int32), np.array([0, 2]), np.array([1, 1]), code, point, codelen, D, 1, 1, 1,
                  seed)
    np.testing.assert_allclose(got[0], want0, rtol=1e-6, atol=1e-9)
    np.testing.assert_array_equal(got[1], I.init_syn0(seed, 2, D)[1])          # neu1e of pair 1 is 0


def test_alpha_schedule(monkeypatch):
    lr = 0.025
    assert I.alpha_at(lr, 1, 10001, 1, 100000, 1) == lr * (1 - 10001 / 100001)
    assert I.alpha_at(lr, 3, 10001, 2, 100000, 4) == lr * (1 - (3 * 10001 + 100000) / 400001)
    assert I.alpha_at(lr, 1, 10 ** 9, 1, 100, 1) == lr * 0.0001                 # the floor
    seen = []
    monkeypatch.setattr(I, "train_pair", lambda s0, s1, last, word, code, point, codelen, alpha, exp, m1:
                        seen.append(alpha))
    n_sent, length = 14, 1000                                   # 14 000 words: one update at the 12th sentence
    words = np.zeros(n_sent * length, np.int32)
    offs = np.arange(0, n_sent * length + 1, length)
    code, point, codelen = I.huffman(np.array([5, 5]))
    words[1::2] = 1
    iters = []
    for k in (1, 2):
        seen.clear()
        I.train_partition(np.zeros((2, 1), np.float32), np.zeros((2, 1), np.float32), np.zeros(2, bool),
                          np.zeros(2, bool), words, offs, range(n_sent), k, 0, 1, 0, 1, 2, len(words), code, point,
                          codelen, I.exp_table())
        iters.append(list(seen))
    for k, a in zip((1, 2), iters):
        assert a[0] == lr                                       # every iteration starts again at lr
        per = 2 * length - 2                                    # pairs per sentence at window 1
        assert set(a[:11 * per]) == {lr}                        # first update once > 10 000 words went by
        assert a[11 * per] == I.alpha_at(lr, 1, 11 * length, k, len(words), 2)
        assert a[-1] == a[11 * per]                             # the next is 10 001 words later


def test_merge_rules():
    glob = np.array([[1, 1], [2, 2], [3, 3]], np.float32)
    local = [np.array([[10, 10], [20, 20], [9, 9]], np.float32), np.array([[7, 7], [30, 31], [8, 8]], np.float32),
             np.array([[5, 5], [40, 41], [6, 6]], np.float32)]
    mod = [np.array([True, True, False]), np.array([False, True, False]), np.array([False, False, False])]
    out = I.merge(glob, local, mod)
    np.testing.assert_array_equal(out[0], local[0][0])                              # one partition: its row
    np.testing.assert_array_equal(out[1], (local[0][1] + local[1][1]) * np.float32(0.5))   # two: the mean
    np.testing.assert_array_equal(out[2], glob[2])                                  # none: the global row
    third = np.float32(1) / np.float32(3)
    mod3 = [np.array([True, False, False])] * 3
    v = np.array([[0.1, 0.7]], np.float32)
    got = I.merge(v, [v * np.float32(k) for k in (1, 2, 3)], [m[:1] for m in mod3])
    np.testing.assert_array_equal(got[0], ((v[0] + v[0] * np.float32(2)) + v[0] * np.float32(3)) * third)


@pytest.mark.parametrize("partitions", [1, 3])
def test_numpy_and_c_oracles_bit_equal(vocab, partitions):
    seqs, ids, counts = vocab
    words, offs = I.chunk_corpus(seqs[:40], ids)
    code, point, codelen = I.huffman(counts)
    args = (words, offs, counts, code, point, codelen, 10, 5, 2, partitions, 7)
    a, b = I.train(*args), X.train(*args)
    assert a.dtype == b.dtype == np.float32
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    assert not np.array_equal(a, I.init_syn0(7, len(counts), 10))


def test_numpy_and_c_oracles_bit_equal_past_the_first_alpha_update():
    """A corpus of more than 10 000 words per partition, one-dimensional vectors: the schedule's update is taken."""
    rng = np.random.default_rng(3)
    counts = np.array([400, 300, 200, 100, 50, 20, 10, 5], np.int64)
    words = rng.integers(0, len(counts), 12000).astype(np.int32)
    offs = np.r_[0, np.arange(700, 12000, 700), 12000]
    code, point, codelen = I.huffman(counts)
    args = (words, offs, counts, code, point, codelen, 1, 1, 2, 1, 5)
    assert np.array_equal(I.train(*args).view(np.int32), X.train(*args).view(np.int32))


def test_user_sums_bit_equal_to_the_shipped_rows():
    r = fixture_ratings()
    sid, svec = shipped_items()
    users, rows, _ = shipped_user_rows()
    ou, ovec = I.user_embeddings(r["userId"], r["movieId"], sid, svec)
    assert np.array_equal(ou, users) and len(users) == 5000
    assert np.array_equal(ovec.view(np.int32), rows.view(np.int32))


def test_writer_reemits_every_shipped_value(tmp_path):
    sid, svec = shipped_items()
    p = tmp_path / "item2vecEmb.csv"
    write_embeddings_csv(str(p), sid, svec)
    with open(os.path.join(GOLDEN, "item2vecEmb.csv")) as f:
        assert p.read_text() == f.read()
    users, rows, lines = shipped_user_rows()
    q = tmp_path / "userEmb.csv"
    write_embeddings_csv(str(q), users, rows)
    assert q.read_text() == "".join(lines)
    back = load_embeddings_csv(str(q))
    assert np.array_equal(back[1].view(np.int32), rows.view(np.int32))


def _raw_item2vec(user, movie, half, ts, D=10, window=5, iters=1, P=1, capacity=16):
    a = [np.ascontiguousarray(x, t) for x, t in ((user, np.int32), (movie, np.int32), (half, np.int8),
                                                 (ts, np.int32))]
    ids = np.zeros(max(capacity, 1), np.int32)
    vec = np.zeros((max(capacity, 1), max(D, 1)), np.float32)
    V = C.c_int32(-1)
    prm = _lib.SrsItem2vecParams(D, window, iters, P, 0)
    rc = _lib.load().srs_item2vec_host(*[x.ctypes.data for x in a], len(a[0]), C.byref(prm), 0, capacity,
                                       ids.ctypes.data, vec.ctypes.data, C.byref(V))
    return rc, V.value


def _raw_users(user, movie, item_ids, D=2, capacity=8):
    u, m, it = (np.ascontiguousarray(x, np.int32) for x in (user, movie, item_ids))
    vec = np.zeros((max(len(it), 1), max(D, 1)), np.float32)
    out_ids = np.zeros(max(capacity, 1), np.int32)
    out = np.zeros((max(capacity, 1), max(D, 1)), np.float32)
    U = C.c_int32(-1)
    rc = _lib.load().srs_user_embeddings_host(u.ctypes.data, m.ctypes.data, len(u), it.ctypes.data, vec.ctypes.data,
                                              len(it), D, 0, capacity, out_ids.ctypes.data, out.ctypes.data,
                                              C.byref(U))
    return rc, U.value


def test_abi_rejections_need_no_device():
    from sparrowrecsys_b200.model import launch_count
    n0 = launch_count()
    u, m, h, t = np.array([1, 1, 2]), np.array([3, 4, 3]), np.array([8, 7, 9]), np.array([5, 6, 7])
    bad = [dict(half=np.array([8, 0, 9])), dict(half=np.array([8, 11, 9])), dict(user=np.array([1, -1, 2])),
           dict(movie=np.array([3, -4, 3])), dict(movie=np.array([3, 1 << 24, 3])), dict(ts=np.array([5, 0, 7])),
           dict(D=0), dict(D=65), dict(window=0), dict(iters=0), dict(P=0), dict(P=(1 << 16) + 1),
           dict(capacity=-1), dict(user=np.zeros(0), movie=np.zeros(0), half=np.zeros(0), ts=np.zeros(0))]
    for b in bad:
        kw = dict(user=u, movie=m, half=h, ts=t)
        kw.update(b)
        rc, V = _raw_item2vec(kw.pop("user"), kw.pop("movie"), kw.pop("half"), kw.pop("ts"), **kw)
        assert rc == _lib.SRS_ERR_INVALID and V == 0, b
    for args, kw in (((u, m, [3, 3]), {}), ((u, m, [-1]), {}), ((u, m, [1 << 24]), {}),
                     ((np.array([1, -2, 2]), m, [3]), {}), ((u, m, [3]), dict(D=0)), ((u, m, [3]), dict(D=65)),
                     ((u, m, [3]), dict(capacity=-1))):
        rc, U = _raw_users(*args, **kw)
        assert rc == _lib.SRS_ERR_INVALID and U == 0, (args, kw)
    assert launch_count() == n0
    msg = _lib.load().srs_last_error().decode()
    assert "capacity" in msg
