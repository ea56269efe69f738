"""DeepWalk graph embedding and the bucketed random-projection LSH on the device (`embedding`, csrc/graphemb.cu,
csrc/lsh.cu) against the numpy oracles (oracle/graphemb.py, oracle/lsh.py) and the C Word2Vec oracle."""
import numpy as np
import pytest

from oracle import graphemb as G
from oracle import item2vec as I
from oracle import item2vec_cext as X
from oracle import lsh as H
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import embedding as E
from sparrowrecsys_b200.model import launch_count

from test_item2vec_oracle import corpus_ratings, fixture_ratings, halves, shipped_items

pytestmark = pytest.mark.gpu


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype.itemsize == b.dtype.itemsize, (a.shape, b.shape, a.dtype, b.dtype)
    bad = np.flatnonzero(a.view(np.uint8).ravel() != b.view(np.uint8).ravel())
    assert bad.size == 0, (bad[:5],)


def _oracle_transitions(r):
    _, seqs = I.positive_sequences(r["userId"], r["movieId"], halves(r), r["timestamp"])
    return G.transitions(seqs)


@pytest.fixture(scope="module")
def ref():
    r = corpus_ratings()
    return r, _oracle_transitions(r)


def test_transitions_exact_on_the_reference_corpus(ref):
    r, tr = ref
    dev = E.item_transitions(r)
    assert len(dev["sources"]) == 956 and len(dev["targets"]) == 124798
    for k in ("sources", "out", "row_ptr", "targets", "counts"):
        assert np.array_equal(dev[k], tr[k]), k
    _bits_equal(dev["dist"], tr["dist"])
    _bits_equal(dev["probs"], tr["probs"])


@pytest.mark.parametrize("seed", [0, 5])
def test_walks_bit_equal_at_the_scripts_size(ref, seed):
    r, tr = ref
    w, n = E.random_walks(r, 20000, 10, seed=seed)
    ow, on = G.random_walks(tr, 20000, 10, seed=seed)
    assert np.array_equal(n, on) and np.array_equal(w, ow)
    assert n.min() >= 1


@pytest.mark.parametrize("W,L", [(3000, 1), (3000, 2), (2000, 1000)])
def test_walk_lengths_bit_equal(ref, W, L):
    r, tr = ref
    w, n = E.random_walks(r, W, L, seed=3)
    ow, on = G.random_walks(tr, W, L, seed=3)
    assert np.array_equal(n, on) and np.array_equal(w, ow)


def _sink_ratings():
    """Chains 1 -> 2 -> 3 and 1 -> 4 (3 and 4 are sinks), 10 -> 11 -> 10, plus non-positive ratings."""
    rows = []
    for u in range(40):
        seq = [1, 2, 3] if u % 3 else [1, 4]
        if u % 5 == 0:
            seq = [10, 11, 10, 11]
        rows += [(u, m, 8, 1000000000 + i) for i, m in enumerate(seq)]
        rows.append((u, 99, 3, 1000000100))               # rated 1.5: not a word
    u, m, h, t = (np.array(c) for c in zip(*rows))
    return {"userId": u.astype(np.int32), "movieId": m.astype(np.int32), "rating": h / 2.0,
            "timestamp": t.astype(np.int32)}


def test_a_graph_with_sinks():
    r = _sink_ratings()
    tr = _oracle_transitions(r)
    assert set(tr["sources"].tolist()) == {1, 2, 10, 11}
    w, n = E.random_walks(r, 500, 6, seed=2)
    ow, on = G.random_walks(tr, 500, 6, seed=2)
    assert np.array_equal(n, on) and np.array_equal(w, ow)
    ends = w[np.arange(len(n)), n - 1]
    assert set(ends[n < 6].tolist()) <= {3, 4}
    dev = E.item_transitions(r)
    assert dev["sources"].tolist() == tr["sources"].tolist() and np.array_equal(dev["probs"], tr["probs"])


def _graph_oracle(r, vector_size, window, iterations, partitions, seed, num_walks, walk_length):
    return G.graph_embedding(r["userId"], r["movieId"], halves(r), r["timestamp"], vector_size, window, iterations,
                             partitions, seed, num_walks, walk_length)


@pytest.mark.parametrize("P", [1, 3])
@pytest.mark.parametrize("D", [10, 33])
def test_graph_embedding_bit_equal_to_the_c_oracle(ref, P, D):
    r, _ = ref
    ids, vec = E.graph_embedding(r, vector_size=D, num_iterations=2, num_partitions=P, seed=4, num_walks=3000,
                                 walk_length=10)
    oids, ovec = _graph_oracle(r, D, 5, 2, P, 4, 3000, 10)
    assert np.array_equal(ids, oids.astype(np.int32))
    _bits_equal(vec, ovec)


def test_graph_embedding_scripts_full_configuration(ref):
    r, _ = ref
    ids, vec = E.graph_embedding(r)
    oids, ovec = _graph_oracle(r, 10, 5, 10, 1, 0, 20000, 10)
    assert np.array_equal(ids, oids.astype(np.int32))
    _bits_equal(vec, ovec)
    assert vec.shape[1] == 10 and len(ids) > 500


def test_graph_embedding_repeat_runs_give_the_same_bits(ref):
    r, _ = ref
    a = E.graph_embedding(r, num_iterations=1, num_partitions=7, num_walks=2000, seed=9)
    b = E.graph_embedding(r, num_iterations=1, num_partitions=7, num_walks=2000, seed=9)
    _bits_equal(a[1], b[1])
    assert np.array_equal(a[0], b[0])
    w1 = E.random_walks(r, 5000, 10, seed=1)
    w2 = E.random_walks(r, 5000, 10, seed=1)
    assert np.array_equal(w1[0], w2[0])


def test_graph_embedding_rejections():
    r = _sink_ratings()
    n0 = launch_count()
    with pytest.raises(ValueError):
        E.graph_embedding(r, num_walks=0)
    assert launch_count() == n0
    # four movies in walks too short for minCount 5: rejected after the counting step
    with pytest.raises(_lib.SrsInvalidError, match="occurrences in the walks"):
        E.graph_embedding({k: v[:3] for k, v in r.items()}, num_walks=1, walk_length=3)


# ---- LSH --------------------------------------------------------------------------------------------------------

def test_lsh_on_the_shipped_vectors():
    sid, svec = shipped_items()
    assert len(sid) == 881
    model = E.BucketedRandomProjectionLSH().fit(svec)
    uv = H.fit(10, 3)
    assert np.array_equal(model.rand_unit_vectors, uv)
    _bits_equal(model.transform(svec), H.transform(svec, uv, 0.1))
    ids, d = model.approx_nearest_neighbors(sid, svec, E.LSH_SAMPLE_KEY, 5)
    oids, od = H.approx_nearest_neighbors(sid, svec, uv, 0.1, E.LSH_SAMPLE_KEY, 5)
    assert len(ids) == 5 and np.array_equal(ids, oids)
    _bits_equal(d, od)
    # every movie as a key, in one call
    res = model.approx_nearest_neighbors(sid, svec, svec.astype(np.float64), 10)
    for q in (0, 1, 440, 880):
        oi, o_d = H.approx_nearest_neighbors(sid, svec, uv, 0.1, svec[q].astype(np.float64), 10)
        assert np.array_equal(res[q][0], oi) and np.array_equal(res[q][1], o_d)
        assert res[q][0][0] == sid[q] and res[q][1][0] == 0.0


@pytest.mark.parametrize("D", [1, 10, 64])
@pytest.mark.parametrize("L", [1, 3, 8])
def test_lsh_on_random_vectors(D, L):
    rng = np.random.default_rng(D * 10 + L)
    n = 4000
    x = rng.standard_normal((n, D)).astype(np.float32)
    ids = rng.permutation(n * 3)[:n].astype(np.int32)
    x[5] = x[6]                                           # a planted distance tie
    bl = 0.5
    model = E.BucketedRandomProjectionLSH(bucket_length=bl, num_hash_tables=L, seed=D + L).fit(x)
    uv = H.fit(D, L, seed=D + L)
    assert np.array_equal(model.rand_unit_vectors, uv)
    _bits_equal(model.transform(x), H.transform(x, uv, bl))
    keys = np.r_[x[:12].astype(np.float64), rng.standard_normal((8, D)) * 0.7, np.full((1, D), 40.0)]
    k = 256 if D == 10 else 20
    batched = model.approx_nearest_neighbors(ids, x, keys, k)
    for q in range(len(keys)):
        single = model.approx_nearest_neighbors(ids, x, keys[q], k)
        oi, od = H.approx_nearest_neighbors(ids, x, uv, bl, keys[q], k)
        assert np.array_equal(batched[q][0], single[0]) and np.array_equal(batched[q][1], single[1])
        assert np.array_equal(single[0], oi), q
        _bits_equal(single[1], od)
    assert len(batched[-1][0]) == len(H.approx_nearest_neighbors(ids, x, uv, bl, keys[-1], k)[0])


def test_lsh_repeat_runs_and_rejections():
    sid, svec = shipped_items()
    model = E.BucketedRandomProjectionLSH().fit(svec)
    a = model.approx_nearest_neighbors(sid, svec, svec[:50].astype(np.float64), 7)
    b = model.approx_nearest_neighbors(sid, svec, svec[:50].astype(np.float64), 7)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a, b))
    n0 = launch_count()
    with pytest.raises(ValueError):
        model.approx_nearest_neighbors(sid, svec, np.zeros(9), 5)
    with pytest.raises(ValueError):
        model.approx_nearest_neighbors(sid, svec, E.LSH_SAMPLE_KEY, 257)
    assert launch_count() == n0


def test_the_command_writes_the_graph_embedding(tmp_path, capsys):
    r = fixture_ratings()
    path = tmp_path / "ratings.csv"
    with open(path, "w") as f:
        f.write("userId,movieId,rating,timestamp\n")
        for row in zip(r["userId"][:20000].tolist(), r["movieId"][:20000].tolist(), r["rating"][:20000].tolist(),
                       r["timestamp"][:20000].tolist()):
            f.write("%d,%d,%s,%d\n" % row)
    assert E.main([str(path), str(tmp_path / "out"), "--graph", "--lsh"]) == 0
    out = capsys.readouterr().out
    assert out.count("Approximately searching for 5 nearest neighbors") == 2
    from sparrowrecsys_b200.ranking import load_embeddings_csv
    ids, vec = load_embeddings_csv(str(tmp_path / "out" / "itemGraphEmb.csv"))
    sub = {k: v[:20000] for k, v in r.items()}
    gids, gvec = E.graph_embedding(sub)
    assert np.array_equal(ids, gids)
    _bits_equal(vec, gvec)
    assert (tmp_path / "out" / "item2vecEmb.csv").exists() and (tmp_path / "out" / "userEmb.csv").exists()
