"""The DeepWalk and LSH oracles (oracle/graphemb.py, oracle/lsh.py) on hand-built cases, known answers and the
reference's corpus, and the device-free rejections of their library entry points.  DESIGN.md section 4.14."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest

from oracle import graphemb as G
from oracle import item2vec as I
from oracle import lsh as H
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import embedding as E

from test_item2vec_oracle import corpus


def _seqs(*rows):
    return [np.asarray(r, np.int64) for r in rows]


def _forced(us):
    """uniforms(w, t) that gives every walk the draw us[t]."""
    return lambda w, t: np.full(len(np.atleast_1d(w)), us[t], np.float64)


# ---- transitions ----------------------------------------------------------------------------------------------------

def test_single_edge_and_a_sink():
    tr = G.transitions(_seqs([3, 7]))
    assert tr["sources"].tolist() == [3] and tr["targets"].tolist() == [7]
    assert tr["probs"].tolist() == [1.0] and tr["dist"].tolist() == [1.0] and tr["row_ptr"].tolist() == [0, 1]
    walks, lengths = G.random_walks(tr, 4, 5, seed=1)
    assert np.all(walks[:, :2] == [3, 7]) and np.all(walks[:, 2:] == -1) and lengths.tolist() == [2] * 4


def test_sentences_of_one_word_have_no_pairs():
    tr = G.transitions(_seqs([5], [6]))
    assert len(tr["sources"]) == 0 and len(tr["targets"]) == 0
    walks, lengths = G.random_walks(tr, 3, 4)
    assert np.all(walks == -1) and np.all(lengths == 0)


def test_out_degree_ten_of_equal_counts():
    tr = G.transitions(_seqs(*[[1, b] for b in range(20, 10, -1)]))
    assert tr["targets"].tolist() == list(range(11, 21)) and tr["counts"].tolist() == [1] * 10
    assert np.all(tr["probs"] == 0.1)
    assert tr["cum"].tolist() == list(itertools.accumulate([0.1] * 10))
    assert tr["cum"][-1] == 1 - 2.0 ** -53                      # ten 0.1s added left to right stay below 1 ...
    walks, lengths = G.random_walks(tr, 1, 2, uniforms=_forced([0.5, 1 - 2.0 ** -53]))
    assert walks[0].tolist() == [1, 20]                          # ... but the largest draw still reaches them
    # u equal to a cumulative sum picks that entry (>=), just above it the next
    c3 = tr["cum"][2]
    assert G.random_walks(tr, 1, 2, uniforms=_forced([0.0, c3]))[0][0].tolist() == [1, 13]
    assert G.random_walks(tr, 1, 2, uniforms=_forced([0.0, np.nextafter(c3, 1)]))[0][0].tolist() == [1, 14]


def test_a_row_draw_past_the_last_sum_repeats_the_current_item():
    tr = G.transitions(_seqs(*[[1, b] for b in range(11, 18)]))
    assert tr["cum"][-1] == 1 - 2 * 2.0 ** -53                  # seven sevenths
    walks, lengths = G.random_walks(tr, 1, 3, uniforms=_forced([0.5, 1 - 2.0 ** -53, 0.0]))
    assert walks[0].tolist() == [1, 1, 11] and lengths[0] == 3


def test_first_draw_past_the_last_sum_gives_an_empty_walk():
    tr = G.transitions(_seqs(*[[a, 100] for a in range(7)]))
    assert tr["cdf"][-1] == 1 - 2 * 2.0 ** -53
    walks, lengths = G.random_walks(tr, 2, 4, uniforms=_forced([1 - 2.0 ** -53, 0.0, 0.0, 0.0]))
    assert np.all(lengths == 0) and np.all(walks == -1)
    assert G.walk_sentences(walks, lengths) == []


def test_walk_lengths_one_and_two():
    tr = G.transitions(_seqs([1, 2, 3, 1]))
    w1, l1 = G.random_walks(tr, 50, 1, seed=3)
    assert np.all(l1 == 1) and set(w1[:, 0].tolist()) <= {1, 2, 3}
    w2, l2 = G.random_walks(tr, 50, 2, seed=3)
    assert np.array_equal(w2[:, 0], w1[:, 0]) and np.all(l2 == 2)
    nxt = {1: 2, 2: 3, 3: 1}
    assert all(nxt[a] == b for a, b in w2.tolist())


def test_walk_draws_and_the_dist_rule():
    tr = G.transitions(_seqs([1, 2, 1, 3], [2, 1]))
    assert tr["sources"].tolist() == [1, 2]                     # 3 is a sink
    assert tr["out"].tolist() == [2, 2] and tr["dist"].tolist() == [0.5, 0.5]
    u = G.walk_uniforms(7, np.arange(5), 2)
    assert np.all((u >= 0) & (u < 1)) and len(set(u.tolist())) == 5
    root = I.splitmix(~7 & ((1 << 64) - 1), 0)
    want = (I.splitmix(I.splitmix(root, 3), 2) >> 11) * 2.0 ** -53
    assert u[3] == want
    assert not np.array_equal(G.walk_uniforms(7, np.arange(5), 1), u)


def test_empirical_transition_frequencies_lie_within_a_binomial_bound():
    rng = np.random.default_rng(5)
    seqs = [rng.integers(0, 12, rng.integers(2, 30)) for _ in range(300)]
    tr = G.transitions(seqs)
    walks, lengths = G.random_walks(tr, 20000, 8, seed=11)
    obs = {}
    for row, n in zip(walks.tolist(), lengths.tolist()):
        for a, b in zip(row[:n - 1], row[1:n]):
            obs.setdefault(a, []).append(b)
    checked = 0
    for r, a in enumerate(tr["sources"].tolist()):
        got = np.asarray(obs.get(a, []))
        if len(got) < 500:
            continue
        lo, hi = tr["row_ptr"][r], tr["row_ptr"][r + 1]
        for b, p in zip(tr["targets"][lo:hi].tolist(), tr["probs"][lo:hi].tolist()):
            f = float(np.mean(got == b))
            assert abs(f - p) <= 5 * math.sqrt(p * (1 - p) / len(got)) + 1e-12, (a, b, f, p)
            checked += 1
    assert checked > 50
    first = np.bincount(np.searchsorted(tr["sources"], walks[:, 0]), minlength=len(tr["sources"])) / len(walks)
    assert np.all(np.abs(first - tr["dist"]) <= 5 * np.sqrt(tr["dist"] * (1 - tr["dist"]) / len(walks)) + 1e-12)


def test_reference_corpus_pins():
    movie, _, off = corpus()
    seqs = [movie[a:b] for a, b in zip(off[:-1], off[1:])]
    a, b = G.pairs(seqs)
    tr = G.transitions(seqs)
    assert len(a) == 627694 and len(tr["targets"]) == 124798
    assert len(tr["sources"]) == 956 and len(np.unique(movie)) == 959       # both sizes graphEmb prints
    assert not np.any(a == b)
    assert int(tr["counts"].sum()) == 627694 and int(tr["out"].sum()) == 627694
    # np.cumsum adds left to right, as the device and the reference do
    assert np.array_equal(tr["cdf"], np.array(list(itertools.accumulate(tr["dist"].tolist()))))
    for lo, hi in zip(tr["row_ptr"][:-1].tolist(), tr["row_ptr"][1:].tolist()):
        assert tr["cum"][hi - 1] == list(itertools.accumulate(tr["probs"][lo:hi].tolist()))[-1]


# ---- java.util.Random and LSH ---------------------------------------------------------------------------------------

def test_java_random_known_answers_and_default_seed():
    assert H.JavaRandom(0).next_int() == -1155484576
    assert H.JavaRandom(42).next_int() == -1170105035
    assert H.DEFAULT_SEED == 772209414 == E.LSH_DEFAULT_SEED
    r = H.JavaRandom(3)
    g = [r.next_gaussian() for _ in range(4)]
    p = E._JavaRandom(3)
    assert g == [p.next_gaussian() for _ in range(4)]         # the library's fit draws the same numbers
    assert all(0 <= H.JavaRandom(s).next_double() < 1 for s in range(20))


def test_fit_gives_unit_vectors_and_matches_the_library():
    uv = H.fit(10, 3)
    assert uv.shape == (3, 10) and np.allclose(np.linalg.norm(uv, axis=1), 1, atol=1e-15)
    lib = E.BucketedRandomProjectionLSH().fit(np.zeros((2, 10), np.float32)).rand_unit_vectors
    assert np.array_equal(lib, uv)
    assert not np.array_equal(H.fit(10, 3, seed=1), uv)


def _uv(rows):
    return np.asarray(rows, np.float64)


def test_lsh_key_with_no_candidates():
    uv = _uv([[1.0, 0.0]])
    x = np.array([[0.0, 0.0], [0.05, 1.0]], np.float32)
    ids, d = H.approx_nearest_neighbors([1, 2], x, uv, 0.1, [5.0, 0.0], 5)
    assert len(ids) == 0 and len(d) == 0


def test_lsh_ties_and_fewer_than_k_candidates():
    uv = _uv([[1.0, 0.0], [0.0, 1.0]])
    x = np.array([[0.01, 0.5], [0.01, -0.5], [0.02, 0.0], [9.0, 9.0]], np.float32)
    ids, d = H.approx_nearest_neighbors([30, 10, 20, 40], x, uv, 0.1, [0.0, 0.0], 5)
    assert ids.tolist() == [20, 10, 30] and d[1] == d[2]          # the tie goes to the lower id


def test_lsh_a_candidate_matching_in_one_table_only():
    uv = _uv([[1.0, 0.0], [0.0, 1.0]])
    x = np.array([[0.05, 3.0], [3.0, 3.0]], np.float32)
    b = H.transform(x, uv, 0.1)
    kb = H.transform(np.array([[0.0, 0.0]]), uv, 0.1)[0]
    assert b[0, 0] == kb[0] and b[0, 1] != kb[1]
    ids, _ = H.approx_nearest_neighbors([1, 2], x, uv, 0.1, [0.0, 0.0], 5)
    assert ids.tolist() == [1]


def test_transform_floors_and_sums_from_zero():
    uv = _uv([[1.0, -1.0]])
    b = H.transform(np.array([[0.25, 0.25], [-0.05, 0.0]], np.float32), uv, 0.1)
    assert b[0, 0] == 0.0 and not np.signbit(b[0, 0]) and b[1, 0] == -1.0


# ---- the library's rejections, before any device call --------------------------------------------------------------

def _ratings():
    u, m, h, t = np.array([1, 1, 2]), np.array([3, 4, 3]), np.array([8, 7, 9]), np.array([5, 6, 7])
    return [np.ascontiguousarray(x, d) for x, d in ((u, np.int32), (m, np.int32), (h, np.int8), (t, np.int32))]


def test_abi_rejections_need_no_device():
    from sparrowrecsys_b200.model import launch_count
    lib = _lib.load()
    n0 = launch_count()
    r = _ratings()
    p = [x.ctypes.data for x in r]
    walks, lengths = np.zeros(100, np.int32), np.zeros(100, np.int32)
    for W, L in ((0, 5), (5, 0), (21000001, 1), (4583, 4583)):
        assert lib.srs_random_walks_host(*p, 3, W, L, 0, 0, walks.ctypes.data, lengths.ctypes.data) \
            == _lib.SRS_ERR_INVALID, (W, L)
    bad_half = np.array([8, 0, 9], np.int8)
    assert lib.srs_random_walks_host(p[0], p[1], bad_half.ctypes.data, p[3], 3, 2, 2, 0, 0, walks.ctypes.data,
                                     lengths.ctypes.data) == _lib.SRS_ERR_INVALID
    ids, vec, V = np.zeros(8, np.int32), np.zeros((8, 10), np.float32), C.c_int32(-1)
    for prm, W in ((_lib.SrsItem2vecParams(0, 5, 1, 1, 0), 10), (_lib.SrsItem2vecParams(10, 5, 1, 1, 0), 0)):
        assert lib.srs_graph_embedding_host(*p, 3, C.byref(prm), W, 10, 0, 8, ids.ctypes.data, vec.ctypes.data,
                                            C.byref(V)) == _lib.SRS_ERR_INVALID
        assert V.value == 0
    S, Ed = C.c_int32(-1), C.c_int32(-1)
    z = np.zeros(8, np.float64)
    assert lib.srs_item_transitions_host(*p, 0, 0, -1, 8, None, None, None, None, walks.ctypes.data,
                                         walks.ctypes.data, z.ctypes.data, C.byref(S), C.byref(Ed)) \
        == _lib.SRS_ERR_INVALID
    x = np.zeros((4, 3), np.float32)
    uv = np.ones((2, 3))
    out = np.zeros((4, 2))
    T = lib.srs_lsh_transform_host
    assert T(x.ctypes.data, 4, 3, uv.ctypes.data, 2, 0.0, 0, out.ctypes.data) == _lib.SRS_ERR_INVALID
    assert T(x.ctypes.data, 4, 3, uv.ctypes.data, 2, float("nan"), 0, out.ctypes.data) == _lib.SRS_ERR_INVALID
    assert T(x.ctypes.data, 4, 3, uv.ctypes.data, 0, 0.1, 0, out.ctypes.data) == _lib.SRS_ERR_INVALID
    assert T(x.ctypes.data, 4, 0, uv.ctypes.data, 2, 0.1, 0, out.ctypes.data) == _lib.SRS_ERR_INVALID
    xn = x.copy()
    xn[2, 1] = np.inf
    assert T(xn.ctypes.data, 4, 3, uv.ctypes.data, 2, 0.1, 0, out.ctypes.data) == _lib.SRS_ERR_INVALID
    key = np.zeros((1, 3))
    oi, od, oc = np.zeros(300, np.int32), np.zeros(300), np.zeros(1, np.int32)
    i4 = np.arange(4, dtype=np.int32)
    Qy = lib.srs_lsh_query_host
    for k in (0, 257):
        assert Qy(i4.ctypes.data, x.ctypes.data, 4, 3, uv.ctypes.data, 2, 0.1, key.ctypes.data, 1, k, 0,
                  oi.ctypes.data, od.ctypes.data, oc.ctypes.data) == _lib.SRS_ERR_INVALID
    keyn = np.array([[0.0, np.nan, 0.0]])
    assert Qy(i4.ctypes.data, x.ctypes.data, 4, 3, uv.ctypes.data, 2, 0.1, keyn.ctypes.data, 1, 5, 0,
              oi.ctypes.data, od.ctypes.data, oc.ctypes.data) == _lib.SRS_ERR_INVALID
    assert launch_count() == n0


def test_python_rejections_need_no_device():
    from sparrowrecsys_b200.model import launch_count
    n0 = launch_count()
    r = {"userId": np.array([1, 1]), "movieId": np.array([3, 4]), "rating": np.array([4.0, 4.0]),
         "timestamp": np.array([5, 6])}
    with pytest.raises(ValueError):
        E.random_walks(r, num_walks=0)
    with pytest.raises(ValueError):
        E.random_walks(r, num_walks=30000, walk_length=1000)
    with pytest.raises(ValueError):
        E.graph_embedding(dict(r, rating=np.array([4.0, 3.3])))
    with pytest.raises(ValueError):
        E.BucketedRandomProjectionLSH(bucket_length=0.0)
    with pytest.raises(ValueError):
        E.BucketedRandomProjectionLSH(num_hash_tables=0)
    m = E.BucketedRandomProjectionLSH().fit(np.zeros((3, 4), np.float32))
    v = np.zeros((3, 4), np.float32)
    with pytest.raises(ValueError):
        m.transform(np.zeros((3, 5), np.float32))                   # dimension mismatch
    with pytest.raises(ValueError):
        m.transform(np.array([[0.1, 0, 0, 0]]))                     # not a float32 value
    with pytest.raises(ValueError):
        m.approx_nearest_neighbors([1, 2, 3], v, np.zeros(5), 3)
    with pytest.raises(ValueError):
        m.approx_nearest_neighbors([1, 2, 3], v, np.array([0, np.inf, 0, 0]), 3)
    with pytest.raises(ValueError):
        m.approx_nearest_neighbors([1, 2, 3], v, np.zeros(4), 0)
    with pytest.raises(ValueError):
        m.approx_nearest_neighbors([1, 2], v, np.zeros(4), 3)
    with pytest.raises(ValueError):
        E.BucketedRandomProjectionLSHModel(np.array([[np.nan, 1.0]]), 0.1)
    assert launch_count() == n0
