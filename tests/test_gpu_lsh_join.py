"""approxSimilarityJoin on the device (`approx_similarity_join`, `srs_lsh_similarity_join_host`, csrc/lsh.cu) against
the oracle (oracle/lsh_join.py): ids, order and distance bits exactly; runs across the join kernel's tile and
segment sizes; one bucket holding every pair; more than 2^31 candidates; the capacity contract; repeat runs and the
documented launch count."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import lsh as H
from oracle import lsh_join as J
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import embedding as E
from sparrowrecsys_b200.model import launch_count

from test_item2vec_oracle import shipped_items

pytestmark = pytest.mark.gpu

_SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc",
                    "lsh.cu")


def _constant(name):
    with open(_SRC) as f:
        return int(eval(re.search(r"constexpr int %s = ([0-9 *]+);" % name, f.read()).group(1)))


# the join kernel's sizes: candidates per tile (threads per block) and segments (blocks) per table
TILE = _constant("kJoinThreads")
SEGMENTS = _constant("kJoinSegments")


def launches(L, pairs_written):
    """lsh.cu's documented count: 3 + 2L when no pair is written (none kept, or more than the capacity), else 4 + 3L."""
    return 4 + 3 * L if pairs_written else 3 + 2 * L


def assert_same(got, want):
    assert got[0].dtype == np.int32 and got[1].dtype == np.int32 and got[2].dtype == np.float64
    assert len(got[0]) == len(want[0]), (len(got[0]), len(want[0]))
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert np.array_equal(got[2].view(np.uint64), np.asarray(want[2], np.float64).view(np.uint64))


def _join_lib(model, ia, xa, ib, xb, threshold, capacity, oa, ob, od):
    P = C.c_int64(-1)
    rc = _lib.load().srs_lsh_similarity_join_host(
        ia.ctypes.data, xa.ctypes.data, len(ia), ib.ctypes.data, xb.ctypes.data, len(ib), model.dim,
        model.rand_unit_vectors.ctypes.data, model.rand_unit_vectors.shape[0], model.bucket_length, threshold, 0,
        capacity, oa.ctypes.data, ob.ctypes.data, od.ctypes.data, C.byref(P))
    return rc, P.value


# ---- the shipped item vectors --------------------------------------------------------------------------------------

@pytest.mark.parametrize("threshold", [0.05, 0.3, 1.0, np.inf])
def test_shipped_vectors_self_join_and_halves(threshold):
    sid, svec = shipped_items()
    model = E.BucketedRandomProjectionLSH().fit(svec)
    uv = H.fit(10, 3)
    n0 = launch_count()
    got = model.approx_similarity_join(sid, svec, sid, svec, threshold)
    assert launch_count() - n0 == launches(3, True)
    assert_same(got, J.approx_similarity_join(sid, svec, sid, svec, uv, 0.1, threshold))
    assert np.sum(got[0] == got[1]) == 881
    a, b = slice(0, 400), slice(881 - 600, 881)
    got = model.approx_similarity_join(sid[a], svec[a], sid[b], svec[b], threshold)
    assert_same(got, J.approx_similarity_join(sid[a], svec[a], sid[b], svec[b], uv, 0.1, threshold))


# ---- random sets ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("D", [1, 10, 64, 1024])
@pytest.mark.parametrize("L", [1, 3, 64])
def test_random_sets(D, L):
    rng = np.random.default_rng(1000 * D + L)
    na, nb = (700, 1100) if D < 1024 else (300, 230)
    xa = rng.standard_normal((na, D)).astype(np.float32)
    xb = np.r_[rng.standard_normal((nb - 20, D)).astype(np.float32), xa[:20]]    # 20 exact copies across sides
    ia = rng.permutation(1 << 20)[:na].astype(np.int32) - (1 << 19)
    ib = rng.permutation(1 << 20)[:nb].astype(np.int32) - (1 << 19)
    bl = {1: 0.05, 10: 0.5, 64: 1.0, 1024: 4.0}[D] * (0.25 if L == 64 else 1.0)
    model = E.BucketedRandomProjectionLSH(bucket_length=bl, num_hash_tables=L, seed=D + L).fit(xa)
    uv = H.fit(D, L, seed=D + L)
    assert np.array_equal(model.rand_unit_vectors, uv)
    every = J.approx_similarity_join(ia, xa, ib, xb, uv, bl, np.inf)
    assert len(every[0]) > 20
    assert_same(model.approx_similarity_join(ia, xa, ib, xb, np.inf), every)
    t = float(np.median(every[2]))
    assert_same(model.approx_similarity_join(ia, xa, ib, xb, t), J.approx_similarity_join(ia, xa, ib, xb, uv, bl, t))
    # B against A: the same pairs swapped, the same distance bits
    ba = model.approx_similarity_join(ib, xb, ia, xa, t)
    fwd = J.approx_similarity_join(ia, xa, ib, xb, uv, bl, t)
    order = np.lexsort((fwd[0], fwd[1]))
    assert_same(ba, (fwd[1][order], fwd[0][order], fwd[2][order]))


def test_an_empty_side_gives_no_pairs_and_no_launch():
    model = E.BucketedRandomProjectionLSH(num_hash_tables=3).fit(np.zeros((1, 8), np.float32))
    x = np.random.default_rng(0).standard_normal((50, 8)).astype(np.float32)
    ids = np.arange(50)
    n0 = launch_count()
    for got in (model.approx_similarity_join([], np.zeros((0, 8), np.float32), ids, x, np.inf),
                model.approx_similarity_join(ids, x, [], np.zeros((0, 8), np.float32), np.inf)):
        assert len(got[0]) == len(got[1]) == len(got[2]) == 0
    assert launch_count() == n0


# ---- runs across the tile and segment sizes --------------------------------------------------------------------------

def _runs_case(run_lengths, filler_total):
    """A dim-1 set per side at bucket length 1 (bucket = floor(x); no value is an integer, so floor(-x) groups the
    rows alike): A row i alone in bucket 3 i against run_lengths[i] B rows, then 400 A rows against
    filler_total // 400 B rows, then filler_total % 400 A rows against one B row, so that the candidates number
    exactly sum(run_lengths) + filler_total."""
    xa, xb = [], []
    for i, n in enumerate(run_lengths):
        k = 3 * i
        xa.append(k + 0.5)
        xb += [k + (j % 127 + 0.5) / 128.0 for j in range(n)]
    base = 3 * len(run_lengths) + 10
    m = 400
    q, extra = divmod(filler_total, m)                   # m rows with q B rows each, plus `extra` singletons
    xa += [base + (j % 97 + 0.5) / 128.0 for j in range(m)]
    xb += [base + (j % 61 + 0.5) / 64.0 for j in range(q)]
    xa += [base + 3 + (j % 89 + 0.5) / 128.0 for j in range(extra)]
    xb += [base + 3.25]
    xa, xb = np.array(xa, np.float32)[:, None], np.array(xb, np.float32)[:, None]
    return xa, xb


@pytest.mark.parametrize("uv", [[[1.0]], [[1.0], [1.0]], [[1.0], [-1.0]]], ids=["L1", "L2same", "L2mirror"])
def test_runs_across_tile_and_segment_sizes(uv):
    S = 300                                              # the segment size made exact: C = S * SEGMENTS
    runs = [S, S - 1, S + 1, TILE - 1, TILE, TILE + 1, 1, 2 * TILE + 1, S + 1, S - 1]
    xa, xb = _runs_case(runs, S * SEGMENTS - sum(runs))
    uv = np.array(uv)
    model = E.BucketedRandomProjectionLSHModel(uv, 1.0)
    ha, hb = H.transform(xa, uv, 1.0), H.transform(xb, uv, 1.0)
    cand = sum(int(np.sum(hb[:, 0] == h)) for h in ha[:, 0])
    assert cand == S * SEGMENTS                          # a second table collides in the same pairs
    rng = np.random.default_rng(3)
    ia = rng.permutation(len(xa) * 2)[:len(xa)].astype(np.int32)
    ib = rng.permutation(len(xb) * 2)[:len(xb)].astype(np.int32)
    for t in (np.inf, 0.3):
        n0 = launch_count()
        got = model.approx_similarity_join(ia, xa, ib, xb, t)
        assert launch_count() - n0 == launches(len(uv), True)
        assert_same(got, J.approx_similarity_join(ia, xa, ib, xb, uv, 1.0, t))
    assert len(got[0]) > 1000


# ---- one bucket ------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def one_bucket():
    rng = np.random.default_rng(7)
    n, D = 3000, 4
    xa = np.abs(rng.standard_normal((n, D))).astype(np.float32)     # every projection >= 0: all in bucket 0
    xb = np.abs(rng.standard_normal((n, D))).astype(np.float32)
    ia = rng.permutation(10 * n)[:n].astype(np.int32) - 5 * n
    ib = rng.permutation(10 * n)[:n].astype(np.int32)
    model = E.BucketedRandomProjectionLSHModel(np.full((1, D), 0.5), 1e30)
    assert np.all(model.transform(xa) == 0.0) and np.all(model.transform(xb) == 0.0)
    oa, ob = np.argsort(ia), np.argsort(ib)
    acc = np.zeros((n, n))
    for d in range(D):
        diff = xa[oa, d].astype(np.float64)[:, None] - xb[ob, d].astype(np.float64)[None, :]
        acc = acc + diff * diff
    want = (np.repeat(ia[oa], n), np.tile(ib[ob], n), np.sqrt(acc).ravel())
    return model, ia, xa, ib, xb, want


def test_one_bucket_gives_every_pair_in_order(one_bucket):
    model, ia, xa, ib, xb, want = one_bucket
    P = 3000 * 3000
    oa, ob, od = np.zeros(P, np.int32), np.zeros(P, np.int32), np.zeros(P)
    rc, n = _join_lib(model, ia, xa, ib, xb, np.inf, P, oa, ob, od)
    assert rc == _lib.SRS_OK and n == P
    assert_same((oa, ob, od), want)


def test_one_bucket_over_capacity_reports_the_size_and_writes_nothing(one_bucket):
    model, ia, xa, ib, xb, want = one_bucket
    P = 3000 * 3000
    oa, ob, od = np.full(P, -77, np.int32), np.full(P, -77, np.int32), np.full(P, -7.5)
    n0 = launch_count()
    rc, n = _join_lib(model, ia, xa, ib, xb, np.inf, P - 1, oa, ob, od)
    assert rc == _lib.SRS_ERR_RANGE and n == P
    assert launch_count() - n0 == launches(1, False)
    assert np.all(oa == -77) and np.all(ob == -77) and np.all(od == -7.5)
    n0 = launch_count()
    got = model.approx_similarity_join(ia, xa, ib, xb, np.inf)     # 2^20 first, then the reported size
    assert launch_count() - n0 == launches(1, False) + launches(1, True)
    assert_same(got, want)


# ---- more than 2^31 candidates ---------------------------------------------------------------------------------------

def test_self_join_of_fifty_thousand_rows_in_one_bucket():
    rng = np.random.default_rng(11)
    n = 50000
    x = rng.random((n, 2)).astype(np.float32)
    assert len(np.unique(x, axis=0)) == n
    ids = rng.permutation(1 << 30)[:n].astype(np.int32)
    model = E.BucketedRandomProjectionLSHModel(np.array([[0.6, 0.8]]), 1e30)
    assert np.all(model.transform(x) == 0.0) and n * n > 2 ** 31     # one bucket: 2.5e9 candidates
    n0 = launch_count()
    ia, ib, d = model.approx_similarity_join(ids, x, ids, x, 1e-300)
    assert launch_count() - n0 == launches(1, True)
    assert np.array_equal(ia, np.sort(ids)) and np.array_equal(ib, ia)
    assert np.all(d == 0.0) and not np.any(np.signbit(d))


# ---- repeat runs, rejections, launches -------------------------------------------------------------------------------

def test_repeat_runs_rejections_and_launch_counts():
    sid, svec = shipped_items()
    model = E.BucketedRandomProjectionLSH(bucket_length=0.3, num_hash_tables=5).fit(svec)
    a = model.approx_similarity_join(sid, svec, sid[::-1], svec[::-1], 0.8)
    b = model.approx_similarity_join(sid, svec, sid[::-1], svec[::-1], 0.8)
    assert_same(a, b)
    assert len(a[0]) > 881
    n0 = launch_count()
    with pytest.raises(ValueError):
        model.approx_similarity_join(np.r_[sid[:-1], sid[:1]], svec, sid, svec, 0.8)
    oa, ob, od = np.zeros(8, np.int32), np.zeros(8, np.int32), np.zeros(8)
    dup = np.r_[sid[:-1], sid[:1]].astype(np.int32)
    x32 = np.ascontiguousarray(svec, np.float32)
    assert _join_lib(model, sid.astype(np.int32), x32, dup, x32, 0.8, 8, oa, ob, od) == (_lib.SRS_ERR_INVALID, -1)
    assert launch_count() == n0
    for t, written in ((0.0, False), (np.nan, False), (-np.inf, False), (0.8, True)):
        n0 = launch_count()
        got = model.approx_similarity_join(sid, svec, sid, svec, t)
        assert launch_count() - n0 == launches(5, written), t
        assert (len(got[0]) > 0) == written
