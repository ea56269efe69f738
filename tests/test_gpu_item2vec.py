"""item2vec and the user embeddings on the device (`embedding`, csrc/item2vec.cu) against the C oracle and the
reference's shipped files."""
import json
import os

import numpy as np
import pytest

from oracle import ctr_oracle as O
from oracle import item2vec as I
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import embedding as E
from sparrowrecsys_b200.model import launch_count
from sparrowrecsys_b200.ranking import rank_by_embedding

from test_item2vec_oracle import (GOLDEN, _raw_item2vec, _raw_users, corpus_ratings, fixture_ratings, halves,
                                  oracle_c, shipped_items, shipped_user_rows)

pytestmark = pytest.mark.gpu


def _same(dev, ref):
    (di, dv), (ri, rv) = dev, ref
    assert np.array_equal(di, ri.astype(np.int32)), (di[:5], ri[:5])
    assert dv.dtype == rv.dtype == np.float32 and dv.shape == rv.shape
    bad = np.flatnonzero(dv.view(np.int32).ravel() != rv.view(np.int32).ravel())
    assert bad.size == 0, (bad[:5], dv.ravel()[bad[:5]], rv.ravel()[bad[:5]])


def _run(r, **kw):
    dev = E.item2vec(r, **kw)
    ref = oracle_c(r, **{{"window_size": "window", "num_iterations": "iterations",
                          "num_partitions": "partitions"}.get(k, k): v for k, v in kw.items()})
    _same(dev, ref)
    return dev


@pytest.fixture(scope="module")
def small():
    return corpus_ratings(users=400)


@pytest.mark.parametrize("partitions", [1, 2, 7, 132, 1000])
def test_partitions_bit_equal_to_the_c_oracle(small, partitions):
    n_sent = 400                                        # no user of the fixture has 1000 positive ratings
    assert partitions != 1000 or partitions > n_sent
    _run(small, vector_size=10, window_size=5, num_iterations=2, num_partitions=partitions, seed=3)


@pytest.mark.parametrize("vector_size", [1, 10, 16, 32, 33, 64])
@pytest.mark.parametrize("window", [1, 5])
def test_vector_sizes_and_windows_bit_equal_to_the_c_oracle(small, vector_size, window):
    _run(small, vector_size=vector_size, window_size=window, num_iterations=2, num_partitions=3, seed=vector_size)


def test_a_user_longer_than_1000_words_is_cut_into_sentences():
    rng = np.random.default_rng(8)
    n_long = 2600
    user = np.r_[np.full(n_long, 7), rng.integers(1, 40, 3000)]
    movie = np.r_[rng.integers(1, 60, n_long), rng.integers(1, 90, 3000)]
    half = np.r_[np.full(n_long, 9), rng.integers(1, 11, 3000)]
    ts = rng.integers(1, 2 ** 31 - 1, len(user))
    r = {"userId": user.astype(np.int32), "movieId": movie.astype(np.int32), "rating": half / 2.0,
         "timestamp": ts.astype(np.int32)}
    _, seqs = I.positive_sequences(user, movie, half, ts)
    assert max(len(s) for s in seqs) > 2000
    for P in (1, 2):
        _run(r, vector_size=12, window_size=5, num_iterations=3, num_partitions=P, seed=1)


@pytest.fixture(scope="module")
def full_run():
    r = corpus_ratings()
    return r, E.item2vec(r, seed=0)


def test_the_scripts_full_run_is_bit_equal_to_the_c_oracle(full_run):
    r, dev = full_run
    _same(dev, oracle_c(r, seed=0))
    _, counts = I.build_vocab(I.positive_sequences(r["userId"], r["movieId"], halves(r), r["timestamp"])[1])
    assert I.huffman(counts)[2].max() >= 15                 # the corpus's deepest path is trained


def test_the_full_run_lies_in_the_recorded_band(full_run):
    import sys
    sys.path.insert(0, GOLDEN)
    from make_item2vec_golden import overlap, top10
    _, (ids, vec) = full_run
    with open(os.path.join(GOLDEN, "item2vec_fit.json")) as f:
        fit = json.load(f)
    sid, svec = shipped_items()
    where = {m: i for i, m in enumerate(ids.tolist())}
    shipped = top10(svec[np.argsort([where[m] for m in sid.tolist()])])
    rec = fit["seeds"]["0"]
    assert overlap(top10(vec), shipped) == pytest.approx(rec["overlap_with_shipped"], abs=1e-12)
    assert float(np.median(np.linalg.norm(vec, axis=1))) == pytest.approx(rec["median_norm"], abs=1e-7)
    assert 1.3 < rec["median_norm"] < 1.7 and abs(fit["shipped_median_norm"] - 1.51) < 0.01


def test_repeat_runs_give_the_same_bits(small):
    for P in (1, 7):
        a = E.item2vec(small, num_iterations=2, num_partitions=P, seed=9)
        b = E.item2vec(small, num_iterations=2, num_partitions=P, seed=9)
        _same(a, b)


def test_user_embeddings_bit_equal_to_the_shipped_rows():
    sid, svec = shipped_items()
    users, rows, _ = shipped_user_rows()
    got = E.user_embeddings(fixture_ratings(), sid, svec)
    _same(got, (users, rows))


def test_find_synonyms_matches_a_numpy_cosine_ranking(full_run):
    _, (ids, vec) = full_run
    sids, sim = E.find_synonyms(ids, vec, 158, 20)
    q = int(np.flatnonzero(ids == 158)[0])
    s = O.cosine_similarity(vec[q], vec).astype(np.float32)
    s[q] = -np.inf
    order = np.argsort(-s.astype(np.float64), kind="stable")[:20]
    assert len(sids) == 20 and 158 not in sids.tolist()
    np.testing.assert_allclose(sim, s[order], atol=1e-6)
    at = np.array([int(np.flatnonzero(ids == x)[0]) for x in sids.tolist()])
    np.testing.assert_allclose(s[at], s[order], atol=1e-6)   # the same ranking up to near-ties


def test_end_to_end_ratings_to_ranked_movies():
    r = fixture_ratings()
    ids, vec = E.item2vec(r, num_iterations=3, seed=4)
    _same((ids, vec), oracle_c(r, iterations=3, seed=4))
    uids, uvec = E.user_embeddings(r, ids, vec)
    ou, ovec = I.user_embeddings(r["userId"], r["movieId"], ids, vec)
    _same((uids, uvec), (ou, ovec))
    for u in (0, 17, len(uids) - 1):
        if not np.any(uvec[u]):
            continue
        pos, top = rank_by_embedding(uvec[u], vec, 10)
        opos, otop = O.rank_topk(O.cosine_similarity(ovec[u], vec).astype(np.float32), 10)
        np.testing.assert_allclose(top, otop, atol=1e-6)
        np.testing.assert_allclose(O.cosine_similarity(ovec[u], vec)[pos], otop, atol=1e-6)


def test_rejections_launch_nothing():
    n0 = launch_count()
    u, m, h, t = np.array([1, 1, 2]), np.array([3, 4, 3]), np.array([8, 7, 9]), np.array([5, 6, 7])
    assert _raw_item2vec(u, m, np.array([8, 0, 9]), t)[0] == _lib.SRS_ERR_INVALID
    assert _raw_item2vec(u, m, h, t, P=0)[0] == _lib.SRS_ERR_INVALID
    assert _raw_users(u, m, [3, 3])[0] == _lib.SRS_ERR_INVALID
    assert launch_count() == n0
    with pytest.raises(ValueError):
        E.item2vec({"userId": u, "movieId": m, "rating": np.array([4.0, 3.3, 5.0]), "timestamp": t})
    assert launch_count() == n0
    # too few ratings for a vocabulary: rejected after the counting step, nothing written
    assert _raw_item2vec(u, m, h, t)[0] == _lib.SRS_ERR_INVALID


def test_the_command_writes_both_files(tmp_path):
    r = fixture_ratings()
    path = tmp_path / "ratings.csv"
    with open(path, "w") as f:
        f.write("userId,movieId,rating,timestamp\n")
        for row in zip(r["userId"][:20000].tolist(), r["movieId"][:20000].tolist(), r["rating"][:20000].tolist(),
                       r["timestamp"][:20000].tolist()):
            f.write("%d,%d,%s,%d\n" % row)
    assert E.main([str(path), str(tmp_path / "out")]) == 0
    from sparrowrecsys_b200.ranking import load_embeddings_csv
    ids, vec = load_embeddings_csv(str(tmp_path / "out" / "item2vecEmb.csv"))
    sub = {k: v[:20000] for k, v in r.items()}
    _same((ids, vec), E.item2vec(sub))
    uids, uvec = load_embeddings_csv(str(tmp_path / "out" / "userEmb.csv"))
    _same((uids, uvec), E.user_embeddings(sub, ids, vec))
