"""approxSimilarityJoin's oracle (oracle/lsh_join.py) against a brute force over every pair, on planted cases and on
the shipped item vectors, and the device-free rejections of `srs_lsh_similarity_join_host` and
`approx_similarity_join`.  DESIGN.md section 4.14."""
import ctypes as C

import numpy as np
import pytest

from oracle import lsh as H
from oracle import lsh_join as J
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import embedding as E
from sparrowrecsys_b200.model import launch_count

from test_item2vec_oracle import shipped_items


def brute_force(ids_a, x_a, ids_b, x_b, uv, bl, threshold):
    """All n_a * n_b pairs at once: a candidate collides in some table; the same sequential distance."""
    xa = np.asarray(x_a, np.float32).astype(np.float64)
    xb = np.asarray(x_b, np.float32).astype(np.float64)
    ha, hb = H.transform(xa, uv, bl), H.transform(xb, uv, bl)
    cand = np.any(ha[:, None, :] == hb[None, :, :], axis=2)
    acc = np.zeros(cand.shape)
    for d in range(xa.shape[1]):
        diff = xa[:, None, d] - xb[None, :, d]
        acc = acc + diff * diff
    dist = np.sqrt(acc)
    a, b = np.nonzero(cand & (dist < threshold))
    ia, ib = np.asarray(ids_a, np.int64)[a], np.asarray(ids_b, np.int64)[b]
    order = np.lexsort((ib, ia))
    return ia[order].astype(np.int32), ib[order].astype(np.int32), dist[a, b][order]


def assert_same(got, want):
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert got[2].dtype == np.float64 and np.array_equal(got[2].view(np.uint64), want[2].view(np.uint64))


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_brute_force_on_random_sets(seed):
    rng = np.random.default_rng(seed)
    D, L = int(rng.integers(1, 9)), int(rng.integers(1, 6))
    na, nb = int(rng.integers(0, 120)), int(rng.integers(1, 150))
    xa = rng.standard_normal((na, D)).astype(np.float32)
    xb = rng.standard_normal((nb, D)).astype(np.float32)
    ia = rng.permutation(1000)[:na].astype(np.int32) - 500
    ib = rng.permutation(1000)[:nb].astype(np.int32) - 500
    uv = H.fit(D, L, seed=seed)
    bl = float(rng.choice([0.3, 1.0, 4.0]))
    for t in (0.5, 2.0, np.inf):
        assert_same(J.approx_similarity_join(ia, xa, ib, xb, uv, bl, t), brute_force(ia, xa, ib, xb, uv, bl, t))


@pytest.mark.parametrize("threshold", [0.05, 0.3, 1.0, np.inf])
def test_oracle_matches_brute_force_on_the_shipped_vectors(threshold):
    sid, svec = shipped_items()
    assert len(sid) == 881
    uv = H.fit(10, 3)
    got = J.approx_similarity_join(sid, svec, sid, svec, uv, 0.1, threshold)
    assert_same(got, brute_force(sid, svec, sid, svec, uv, 0.1, threshold))
    assert len(got[0]) >= 881                                 # every movie with itself
    half = J.approx_similarity_join(sid[:400], svec[:400], sid[-600:], svec[-600:], uv, 0.1, threshold)
    assert_same(half, brute_force(sid[:400], svec[:400], sid[-600:], svec[-600:], uv, 0.1, threshold))


def _two_tables():
    return np.array([[1.0, 0.0], [0.0, 1.0]])


def test_a_pair_colliding_only_in_the_last_table_appears_once():
    uv = _two_tables()
    xa = np.array([[0.5, 0.5]], np.float32)
    xb = np.array([[3.5, 0.25], [0.25, 3.5]], np.float32)     # row 0 collides in table 1 only, row 1 in table 0
    ha, hb = H.transform(xa, uv, 1.0), H.transform(xb, uv, 1.0)
    assert ha[0, 0] != hb[0, 0] and ha[0, 1] == hb[0, 1] and ha[0, 0] == hb[1, 0] and ha[0, 1] != hb[1, 1]
    ia, ib, d = J.approx_similarity_join([7], xa, [1, 2], xb, uv, 1.0, np.inf)
    assert ia.tolist() == [7, 7] and ib.tolist() == [1, 2]


def test_a_pair_colliding_in_every_table_appears_once():
    uv = H.fit(4, 8, seed=3)
    x = np.array([[0.1, 0.2, 0.3, 0.4]], np.float32)
    y = x + np.float32(1e-6)
    assert np.all(H.transform(x, uv, 10.0) == H.transform(y, uv, 10.0))
    ia, ib, d = J.approx_similarity_join([1], x, [2], y, uv, 10.0, 1.0)
    assert ia.tolist() == [1] and ib.tolist() == [2] and 0 < d[0] < 1e-5


def test_a_distance_equal_to_the_threshold_is_excluded():
    uv = np.array([[1.0, 0.0]])
    xa, xb = np.array([[0.0, 0.0]], np.float32), np.array([[3.0, 4.0]], np.float32)
    assert len(J.approx_similarity_join([1], xa, [2], xb, uv, 1e30, 5.0)[0]) == 0
    ia, ib, d = J.approx_similarity_join([1], xa, [2], xb, uv, 1e30, np.nextafter(5.0, np.inf))
    assert ia.tolist() == [1] and ib.tolist() == [2] and d.tolist() == [5.0]


def test_a_self_join_has_self_pairs_and_is_symmetric():
    rng = np.random.default_rng(4)
    x = rng.standard_normal((60, 3)).astype(np.float32)
    ids = rng.permutation(200)[:60].astype(np.int32)
    uv = H.fit(3, 2, seed=1)
    ia, ib, d = J.approx_similarity_join(ids, x, ids, x, uv, 1.0, 1.5)
    selfs = ia == ib
    assert sorted(ia[selfs].tolist()) == sorted(ids.tolist()) and np.all(d[selfs] == 0.0)
    fwd = {(a, b): v for a, b, v in zip(ia.tolist(), ib.tolist(), d.tolist())}
    assert all(fwd[(b, a)] == v for (a, b), v in fwd.items())
    assert len(fwd) > 2 * 60


def test_nan_negative_infinity_and_zero_thresholds_give_nothing():
    sid, svec = shipped_items()
    uv = H.fit(10, 3)
    for t in (np.nan, -np.inf, 0.0, -1.0):
        assert len(J.approx_similarity_join(sid[:100], svec[:100], sid[:100], svec[:100], uv, 0.1, t)[0]) == 0
    assert len(J.approx_similarity_join(sid[:100], svec[:100], sid[:100], svec[:100], uv, 0.1, 5e-324)[0]) == 100


# ---- the library's rejections, before any device call --------------------------------------------------------------

def _join_args(**kw):
    x = np.zeros((4, 3), np.float32)
    a = dict(ids_a=np.arange(4, dtype=np.int32), vectors_a=x, n_a=4, ids_b=np.arange(4, dtype=np.int32) + 10,
             vectors_b=x.copy(), n_b=4, dim=3, uv=np.ones((2, 3)), L=2, bl=0.1, threshold=1.0, device=0,
             capacity=16, oa=np.zeros(16, np.int32), ob=np.zeros(16, np.int32), od=np.zeros(16), n_pairs=C.c_int64(-7))
    a.update(kw)
    p = lambda v: None if v is None else v.ctypes.data
    args = (p(a["ids_a"]), p(a["vectors_a"]), a["n_a"], p(a["ids_b"]), p(a["vectors_b"]), a["n_b"], a["dim"],
            p(a["uv"]), a["L"], a["bl"], a["threshold"], a["device"], a["capacity"], p(a["oa"]), p(a["ob"]),
            p(a["od"]), None if a["n_pairs"] is None else C.byref(a["n_pairs"]))
    return args, a["n_pairs"]


def _last_error():
    return _lib.load().srs_last_error().decode()


def test_abi_rejections_need_no_device():
    lib = _lib.load()
    J_ = lib.srs_lsh_similarity_join_host
    n0 = launch_count()
    dup = np.array([1, 2, 3, 2], np.int32)
    bad_x = np.zeros((4, 3), np.float32)
    bad_x[1, 2] = np.nan
    inf_x = np.zeros((4, 3), np.float32)
    inf_x[3, 0] = -np.inf
    nan_uv = np.ones((2, 3))
    nan_uv[1, 1] = np.nan
    cases = [dict(ids_a=dup), dict(ids_b=dup), dict(dim=0), dict(dim=1025), dict(L=0), dict(L=65),
             dict(vectors_a=bad_x), dict(vectors_b=inf_x), dict(uv=nan_uv), dict(bl=0.0), dict(bl=-0.1),
             dict(bl=np.nan), dict(bl=np.inf), dict(n_a=-1), dict(n_b=-1), dict(n_a=1 << 31), dict(capacity=-1),
             dict(n_pairs=None), dict(oa=None), dict(ob=None), dict(od=None), dict(ids_a=None), dict(ids_b=None),
             dict(vectors_a=None), dict(vectors_b=None), dict(uv=None)]
    for kw in cases:
        args, n_pairs = _join_args(**kw)
        assert J_(*args) == _lib.SRS_ERR_INVALID, kw
        if n_pairs is not None:
            assert n_pairs.value == -7, kw                         # nothing written on a rejection
    args, _ = _join_args(ids_a=dup)
    J_(*args)
    assert "ids_a" in _last_error() and "id 2" in _last_error()
    args, _ = _join_args(ids_b=np.array([-5, 9, -5, 0], np.int32))
    J_(*args)
    assert "ids_b" in _last_error() and "id -5" in _last_error()
    # capacity 0 needs no outputs; an empty side returns no pairs without touching the device
    for kw in (dict(n_a=0), dict(n_b=0), dict(n_a=0, capacity=0, oa=None, ob=None, od=None)):
        args, n_pairs = _join_args(**kw)
        assert J_(*args) == _lib.SRS_OK and n_pairs.value == 0, kw
    assert launch_count() == n0


def test_python_rejections_need_no_device():
    n0 = launch_count()
    m = E.BucketedRandomProjectionLSH().fit(np.zeros((3, 4), np.float32))
    v = np.zeros((3, 4), np.float32)
    i3 = np.array([1, 2, 3])
    with pytest.raises(ValueError, match="ids_a"):
        m.approx_similarity_join([1, 1, 3], v, i3, v, 1.0)
    with pytest.raises(ValueError, match="ids_b holds id 3"):
        m.approx_similarity_join(i3, v, [3, 2, 3], v, 1.0)
    with pytest.raises(ValueError):
        m.approx_similarity_join([1, 2], v, i3, v, 1.0)           # ids and vectors differ in length
    with pytest.raises(ValueError):
        m.approx_similarity_join(i3, v, i3, np.zeros((3, 5), np.float32), 1.0)   # dimension mismatch
    with pytest.raises(ValueError):
        m.approx_similarity_join(i3, np.array([[0.1, 0, 0, 0]] * 3), i3, v, 1.0)   # not float32 values
    with pytest.raises(ValueError):
        m.approx_similarity_join(i3, v, i3, np.full((3, 4), np.inf, np.float32), 1.0)
    # an empty side: no pairs, no device call
    ia, ib, d = m.approx_similarity_join([], np.zeros((0, 4), np.float32), i3, v, 1.0)
    assert ia.dtype == np.int32 and ib.dtype == np.int32 and d.dtype == np.float64 and len(ia) == len(d) == 0
    assert launch_count() == n0
