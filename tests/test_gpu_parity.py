"""CUDA path vs oracle, through the C ABI (needs a GPU: pytest -m gpu).

Tolerance: BASELINE.json's north_star asks for predictions within 1e-4 of the
reference float32 `model.predict`; these tests hold the CUDA path to PROB_ATOL = 2e-5
on probabilities and LOGIT_ATOL = 2e-4 on logits (logits are O(1..10); comparing them
keeps the check meaningful where the sigmoid saturates).
"""
import numpy as np
import pytest

from conftest import load_golden_weights
from oracle import ctr_oracle as O
from sparrowrecsys_b200.features import encode_batch, synthetic_features
from sparrowrecsys_b200.spec import baseline_spec, default_spec
from sparrowrecsys_b200.weights import init_weights

pytestmark = pytest.mark.gpu

PROB_ATOL = 2e-5
LOGIT_ATOL = 2e-4
MODELS = ["embeddingmlp", "widendeep", "neuralcf", "twotowers", "deepfm", "deepfm_v2", "din"]


def _model(spec, W):
    from sparrowrecsys_b200.model import CTRModel
    return CTRModel(spec, W, device=0)


def _compare(spec, W, feats, prob_atol=PROB_ATOL, logit_atol=LOGIT_ATOL):
    with _model(spec, W) as m:
        p, z = m.predict_with_logits(feats)
    po, zo = O.forward(spec, W, feats)
    assert p.shape == po.shape == (len(feats["movieId"]), 1) and p.dtype == np.float32
    assert np.abs(z - zo).max() <= logit_atol, "logit err %g" % np.abs(z - zo).max()
    assert np.abs(p - po).max() <= prob_atol, "prob err %g" % np.abs(p - po).max()
    return p, z


# ---- golden: shipped trained weights ---------------------------------------------------
def test_neuralcf_shipped_weights_known_answers(head_rows):
    from test_oracle_golden import KNOWN
    W = load_golden_weights("neuralcf_002")
    p, _ = _compare(default_spec("neuralcf"), W, head_rows)
    np.testing.assert_allclose(p[:8, 0], KNOWN["neuralcf_002"], rtol=0, atol=1e-6)
    W1 = load_golden_weights("neuralcf_001")
    p1, _ = _compare(default_spec("neuralcf"), W1, head_rows)
    np.testing.assert_allclose(p1[:8, 0], KNOWN["neuralcf_001"], rtol=0, atol=1e-6)


def test_twotowers_shipped_weights_known_answers(head_rows):
    from test_oracle_golden import KNOWN
    W = load_golden_weights("mlprec_005")
    spec = default_spec("twotowers", hidden=(10,), final_dense=False)
    p, z = _compare(spec, W, head_rows)
    np.testing.assert_allclose(p[:8, 0], KNOWN["mlprec_005"], rtol=0, atol=1e-6)
    assert np.array_equal(p, z)


@pytest.mark.parametrize("name", ["neuralcf_002", "neuralcf_001", "mlprec_005"])
def test_shipped_weights_against_the_serialised_serving_graphs(name):
    """CUDA path vs the outputs of the reference's own serialised `serving_default` functions (evaluated node by
    node by oracle/savedmodel_graph.py; tests/golden/savedmodel_graph_vectors.json): 512 head rows + the
    HttpClient pair.  A wiring mistake (concat order, kernel binding, activation) would be an O(0.1) difference."""
    import json
    import os
    from conftest import GOLDEN
    with open(os.path.join(GOLDEN, "savedmodel_graph_vectors.json")) as f:
        v = json.load(f)[name]
    W = load_golden_weights(name)
    feats = {"movieId": np.array(v["movieId"], np.int32), "userId": np.array(v["userId"], np.int32)}
    spec = default_spec("twotowers", hidden=(10,), final_dense=False) if name == "mlprec_005" else default_spec("neuralcf")
    with _model(spec, W) as m:
        p = m.predict(feats)
    np.testing.assert_allclose(p[:, 0], np.array(v["output"], np.float32), rtol=0, atol=PROB_ATOL)


def test_httpclient_pair_through_tfrecmodel_surface():
    from tfrecmodel import neuralcf
    neuralcf.load(weights=load_golden_weights("neuralcf_002"))
    p = neuralcf.predict({"userId": np.array([10351, 10351]), "movieId": np.array([52, 53])})
    np.testing.assert_allclose(p[:, 0], [0.68536943, 0.17321654], rtol=0, atol=1e-6)
    assert p.shape == (2, 1) and p.dtype == np.float32
    neuralcf.model.close()


# ---- every model, reference shapes, real rows ------------------------------------------
@pytest.mark.parametrize("model", MODELS)
def test_reference_shape_on_bundled_rows(model, head_rows):
    spec = default_spec(model)
    _compare(spec, init_weights(spec, 100 + MODELS.index(model)), head_rows)


def test_twotowers_with_final_dense_and_deeper_towers(head_rows):
    spec = default_spec("twotowers", hidden=(16, 8), final_dense=True)
    _compare(spec, init_weights(spec, 5), head_rows)
    spec = default_spec("neuralcf", hidden=(32, 16, 8))
    _compare(spec, init_weights(spec, 6), head_rows)


# ---- BASELINE.json shapes (synthetic MovieLens-20M-shaped inputs) -----------------------
@pytest.mark.parametrize("cfg,B,seed", [("cfg2_deepfm", 4096, 1), ("cfg2_deepfm_v2", 4096, 1),
                                        ("cfg3_din", 4096, 2), ("cfg4_widendeep", 8192, 3),
                                        ("cfg4_neuralcf", 8192, 3), ("cfg4_twotowers", 8192, 3)])
def test_baseline_configs(cfg, B, seed):
    spec = baseline_spec(cfg)
    W = init_weights(spec, seed)
    feats = synthetic_features(spec, B, seed=seed)
    _compare(spec, W, feats)


def test_din_long_history_wide_embedding():
    """cfg 5 shape at a vocabulary the oracle can hold: E=64, T=200."""
    spec = default_spec("din", emb_dim=64, hist_len=200, n_movies=200_000, n_users=5000)
    W = init_weights(spec, 4)
    feats = synthetic_features(spec, 512, seed=4, uniform_history=True)
    _compare(spec, W, feats, logit_atol=5e-4)


def test_din_cfg5_at_the_real_vocabulary():
    """BASELINE cfg 5 as stated: V = 10^8 movies, E = 64, T = 200 - a 25.6 GB table generated in place in HBM
    (srs_fill_uniform) and borrowed by the model.  The oracle cannot hold that table: it regenerates exactly the
    rows the batch touches with the same counter-based formula (oracle.fill_uniform), remaps the ids to that
    compact table and runs the reference graph on it."""
    import torch
    from dataclasses import replace
    from sparrowrecsys_b200 import _lib
    from sparrowrecsys_b200.spec import baseline_spec
    free, _ = torch.cuda.mem_get_info(0)
    if free < 70e9:
        pytest.skip("needs ~55 GB of free HBM (25.6 GB table + its pre-split copy)")
    spec = baseline_spec("cfg5_din")
    B = 96
    W = init_weights(spec, 4, skip=("embedding",))
    feats = synthetic_features(spec, B, seed=9, uniform_history=True)
    # DIN.py:95,125: the ids pass through a float32 numeric_column before the Embedding casts them back, so above
    # 2^24 an id selects the row of its float32 rounding (99 999 937 -> 99 999 936); ids that would round to
    # 10^8 = num_buckets are kept out (TF would assert)
    top = 99_999_992
    for k in ["movieId"] + ["userRatedMovie%d" % (t + 1) for t in range(spec.hist_len)]:
        feats[k] = np.minimum(np.asarray(feats[k]), top).astype(np.int32)
    feats["movieId"][:4] = [top, 0, 1, 99_999_937]                       # the ends of the table, an inexact id
    dev = torch.device("cuda", 0)
    table = torch.empty(spec.n_movies, spec.emb_dim, dtype=torch.float32, device=dev)
    _lib.check(_lib.load().srs_fill_uniform(table.data_ptr(), table.numel(), 1234, -0.05, 0.05, 0, None))
    torch.cuda.synchronize()
    Wd = dict(W)
    Wd["embedding"] = table
    with _model(spec, Wd) as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
    del table
    torch.cuda.empty_cache()
    # the oracle side: compact table of the touched rows
    keys = ["movieId"] + ["userRatedMovie%d" % (k + 1) for k in range(spec.hist_len)]
    rt = lambda a: np.asarray(a).astype(np.float32).astype(np.int64)      # the float32 round trip of the graph
    touched = np.unique(np.concatenate([rt(feats[k]) for k in keys]))
    E = spec.emb_dim
    flat = (touched[:, None] * E + np.arange(E)[None, :]).reshape(-1)
    small = replace(spec, n_movies=int(touched.shape[0]))
    Wo = dict(W)
    Wo["embedding"] = O.fill_uniform(flat, 1234, -0.05, 0.05).reshape(-1, E)
    fo = dict(feats)
    for k in keys:
        fo[k] = np.searchsorted(touched, rt(feats[k])).astype(np.int32)
    po, zo = O.forward(small, Wo, fo)
    assert np.abs(z - zo).max() <= 5e-4, "logit err %g" % np.abs(z - zo).max()
    assert np.abs(p - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p - po).max()


@pytest.mark.parametrize("E,T", [(10, 5), (16, 7), (32, 33), (12, 64), (8, 1)])
def test_din_shapes(E, T):
    spec = default_spec("din", emb_dim=E, hist_len=T, n_movies=5000, n_users=3000)
    W = init_weights(spec, E * 100 + T)
    feats = synthetic_features(spec, 333, seed=T)
    _compare(spec, W, feats)


@pytest.mark.parametrize("model", ["embeddingmlp", "deepfm", "deepfm_v2"])
@pytest.mark.parametrize("E", [10, 16, 32])
def test_embedding_widths(model, E):
    spec = default_spec(model, emb_dim=E, n_movies=3000, n_users=4000)
    W = init_weights(spec, E)
    _compare(spec, W, synthetic_features(spec, 777, seed=E))


# ---- edge cases ------------------------------------------------------------------------
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("B", [1, 2, 31, 63, 65, 129])
def test_ragged_batch_sizes(model, B, head_rows):
    spec = default_spec(model)
    W = init_weights(spec, 9)
    sub = {k: v[:B] for k, v in head_rows.items()}
    _compare(spec, W, sub)


def test_empty_batch():
    spec = default_spec("din")
    with _model(spec, init_weights(spec, 0)) as m:
        f = synthetic_features(spec, 4, seed=0)
        p = m.predict({k: v[:0] for k, v in f.items()})
        assert p.shape == (0, 1)


@pytest.mark.parametrize("model", ["embeddingmlp", "widendeep", "deepfm", "deepfm_v2", "din"])
def test_all_genres_missing_and_zero_history(model, head_rows):
    spec = default_spec(model)
    W = init_weights(spec, 21)
    sub = {k: v[:100].copy() for k, v in head_rows.items()}
    for k in list(sub):
        if "Genre" in k:
            sub[k] = np.array([""] * 100, dtype=object)
        if k.startswith("userRatedMovie"):
            sub[k] = np.zeros(100, np.int32)
    _compare(spec, W, sub)


def test_vocabulary_extremes():
    spec = default_spec("din")
    W = init_weights(spec, 22)
    f = synthetic_features(spec, 64, seed=1)
    f["movieId"][:] = spec.n_movies - 1
    f["userId"][:] = spec.n_users - 1
    f["userRatedMovie1"][:] = spec.n_movies - 1
    f["movieId"][::2] = 0
    f["userId"][::2] = 0
    _compare(spec, W, f)


def test_out_of_range_ids_raise_value_error():
    from sparrowrecsys_b200 import _lib
    import ctypes as C
    spec = default_spec("neuralcf")
    with _model(spec, init_weights(spec, 0)) as m:
        with pytest.raises(ValueError):          # host-side check (mirrors TF's assert)
            m.predict({"movieId": np.array([5000]), "userId": np.array([1])})
        # straight through the ABI: the kernel latches the flag, never faults
        enc = encode_batch(spec, {"movieId": np.array([1, 2]), "userId": np.array([1, 2])})
        enc.movie_id[1] = 123456
        out = np.zeros(2, np.float32)
        with pytest.raises(ValueError):
            m.predict_encoded(enc, out)
        enc.movie_id[1] = 2                      # flag is cleared: next call is clean
        m.predict_encoded(enc, out)
        assert np.isfinite(out).all()


def test_missing_key_raises_key_error():
    spec = default_spec("din")
    with _model(spec, init_weights(spec, 0)) as m:
        f = synthetic_features(spec, 4, seed=0)
        del f["userRatedMovie3"]
        with pytest.raises(KeyError):
            m.predict(f)


def test_bad_weights_rejected():
    from sparrowrecsys_b200.model import CTRModel
    spec = default_spec("neuralcf")
    W = init_weights(spec, 0)
    bad = dict(W)
    bad["dense_1/kernel"] = np.zeros((3, 3), np.float32)
    with pytest.raises(ValueError):
        CTRModel(spec, bad)
    del bad["dense_1/kernel"]
    with pytest.raises(KeyError):
        CTRModel(spec, bad)


# ---- device-resident path and size-independent properties at full size ------------------
def test_device_path_matches_host_path_and_is_deterministic():
    import torch
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 2)
    feats = synthetic_features(spec, 4096, seed=2)
    with _model(spec, W) as m:
        p_host = m.predict(feats)[:, 0]
        db = m.to_device(feats)
        out = torch.empty(4096, dtype=torch.float32, device="cuda:0")
        lg = torch.empty_like(out)
        m.predict_device(db, out, lg)
        torch.cuda.synchronize()
        a = out.cpu().numpy().copy()
        m.predict_device(db, out, lg)
        torch.cuda.synchronize()
        assert np.array_equal(a, out.cpu().numpy())          # run-to-run bit identical
        assert np.array_equal(a, p_host)                     # host path == device path
        m.status()


@pytest.mark.parametrize("cfg,B", [("cfg4_widendeep", 65536), ("cfg4_neuralcf", 65536),
                                   ("cfg3_din", 16384)])
def test_row_independence_at_full_size(cfg, B):
    """Rows are independent: scoring a permutation of the batch permutes the scores, and
    scoring two halves separately equals scoring the whole (the sharding invariant),
    bit for bit; a sample of rows is checked against the oracle."""
    spec = baseline_spec(cfg)
    W = init_weights(spec, 3)
    feats = synthetic_features(spec, B, seed=3)
    rng = np.random.default_rng(0)
    perm = rng.permutation(B)
    with _model(spec, W) as m:
        p = m.predict(feats)[:, 0]
        pp = m.predict({k: v[perm] for k, v in feats.items()})[:, 0]
        assert np.array_equal(pp, p[perm])
        half = B // 2 + 17
        lo = m.predict({k: v[:half] for k, v in feats.items()})[:, 0]
        hi = m.predict({k: v[half:] for k, v in feats.items()})[:, 0]
        assert np.array_equal(np.concatenate([lo, hi]), p)
        p12 = m.predict(feats, batch_size=4099)[:, 0]        # Keras-style batched predict
        assert np.array_equal(p12, p)
    idx = rng.choice(B, 512, replace=False)
    po, _ = O.forward(spec, W, {k: v[idx] for k, v in feats.items()})
    assert np.abs(p[idx] - po[:, 0]).max() <= PROB_ATOL
    assert 0.0 < p.min() and p.max() < 1.0 and p.std() > 0.01


def test_pipelined_host_slots_match_sync_path():
    import ctypes as C
    import torch
    from sparrowrecsys_b200 import _lib
    spec = default_spec("din")
    W = init_weights(spec, 8)
    with _model(spec, W) as m:
        n_slots = m.num_slots()
        batches, outs, keeps = [], [], []
        for i in range(2 * n_slots):
            f = synthetic_features(spec, 300 + i, seed=i)
            enc = encode_batch(spec, f)
            pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
            t = dict(movie=pin(enc.movie_id), user=pin(enc.user_id), hist=pin(enc.hist),
                     mg=pin(enc.movie_genre), ug=pin(enc.user_genre), num=pin(enc.numerics),
                     out=torch.empty(enc.B, dtype=torch.float32).pin_memory())
            b = _lib.SrsBatch(enc.B, enc.hist.shape[1], t["movie"].data_ptr(), t["user"].data_ptr(),
                              t["hist"].data_ptr(), t["mg"].data_ptr(), t["ug"].data_ptr(),
                              t["num"].data_ptr())
            keeps.append(t)
            batches.append((f, b, t["out"]))
        for i, (f, b, out) in enumerate(batches):
            slot = i % n_slots
            if i >= n_slots:
                m.wait(slot)
            m.submit_host(slot, b, out.data_ptr())
        for s in range(n_slots):
            m.wait(s)
        for f, b, out in batches:
            ref = m.predict(f)[:, 0]
            assert np.array_equal(out.numpy(), ref)


def test_borrowed_device_table_and_fill_uniform():
    """cfg 5 mechanics at small scale: the movie table is generated in HBM by
    srs_fill_uniform and used in place; the oracle regenerates the rows it needs."""
    import torch
    from sparrowrecsys_b200 import _lib
    from sparrowrecsys_b200.model import CTRModel
    V, E = 50_000, 64
    spec = default_spec("din", emb_dim=E, hist_len=20, n_movies=V, n_users=2000)
    W = init_weights(spec, 4, skip=("embedding",))
    table = torch.empty(V, E, dtype=torch.float32, device="cuda:0")
    lib = _lib.load()
    _lib.check(lib.srs_fill_uniform(table.data_ptr(), V * E, 1234, -0.05, 0.05, 0, None))
    torch.cuda.synchronize()
    host = O.fill_uniform(np.arange(V * E), 1234, -0.05, 0.05).reshape(V, E)
    assert np.array_equal(table.cpu().numpy(), host)          # bit exact generator
    feats = synthetic_features(spec, 256, seed=4, uniform_history=True)
    Wd = dict(W)
    Wd["embedding"] = table
    with CTRModel(spec, Wd) as m:
        p, z = m.predict_with_logits(feats)
    Wh = dict(W)
    Wh["embedding"] = host
    po, zo = O.forward(spec, Wh, feats)
    assert np.abs(p - po).max() <= PROB_ATOL and np.abs(z - zo).max() <= LOGIT_ATOL


def test_cosine_scores():
    import torch
    from sparrowrecsys_b200 import _lib
    rng = np.random.default_rng(0)
    q = rng.standard_normal(10).astype(np.float32)
    c = rng.standard_normal((800, 10)).astype(np.float32)
    dq, dc = torch.from_numpy(q).cuda(), torch.from_numpy(c).cuda()
    out = torch.empty(800, dtype=torch.float32, device="cuda:0")
    _lib.check(_lib.load().srs_cosine_scores_device(dq.data_ptr(), dc.data_ptr(), 800, 10,
                                                    out.data_ptr(), 0, None))
    torch.cuda.synchronize()
    ref = O.cosine_similarity(q, c)
    assert np.abs(out.cpu().numpy() - ref).max() < 1e-6


def test_launch_counter_counts_kernels():
    from sparrowrecsys_b200.model import launch_count
    spec = default_spec("neuralcf")
    with _model(spec, init_weights(spec, 0)) as m:
        before = launch_count()
        m.predict({"movieId": np.array([1, 2, 3]), "userId": np.array([1, 2, 3])})
        assert launch_count() == before + 1


# ---- DIN tensor-core kernel (csrc/din_wg.cu, warpgroup MMAs) vs CUDA-core kernel vs oracle ----
#      sm_cap 0 runs it with one CTA per 32-row tile; sm_cap 7 caps the grid at 7 CTAs, so that every CTA
#      walks several tiles in its grid-stride loop.

@pytest.fixture
def din_impl(monkeypatch):
    def set_impl(name):
        monkeypatch.setenv("SRS_DIN_IMPL", name)
    return set_impl


@pytest.mark.parametrize("E,T,B", [(32, 50, 4096), (32, 9, 100), (32, 31, 17), (32, 32, 16),
                                   (32, 33, 15), (20, 64, 333), (32, 65, 129), (32, 128, 257),
                                   (24, 100, 1), (32, 50, 4097)])
@pytest.mark.parametrize("sm_cap", [0, 7])
def test_din_tensor_core_kernel(E, T, B, sm_cap, din_impl):
    spec = default_spec("din", emb_dim=E, hist_len=T, n_movies=27279, n_users=5000)
    W = init_weights(spec, E * 1000 + T)
    feats = synthetic_features(spec, B, seed=T)
    din_impl("tc")
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        m.set_sm_limit(sm_cap)
        p_tc, z_tc = m.predict_with_logits(feats)
        p_tc2 = m.predict(feats)
    assert np.array_equal(p_tc, p_tc2)                       # deterministic
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z_tc - zo).max() <= LOGIT_ATOL, "logit err %g" % np.abs(z_tc - zo).max()
    assert np.abs(p_tc - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p_tc - po).max()
    din_impl("cudacore")
    with _model(spec, W) as m:
        assert m.kernel_name == "din_kernel"
        p_cc = m.predict(feats)
    assert np.abs(p_cc - po).max() <= PROB_ATOL
    assert np.abs(p_cc - p_tc).max() <= 2 * PROB_ATOL


@pytest.mark.parametrize("E,T,B", [(64, 200, 512), (64, 128, 100), (48, 129, 33), (33, 9, 17), (64, 256, 65),
                                   (40, 64, 4097), (64, 200, 1), (64, 130, 148 * 32 + 5)])
def test_din_row_tile_kernel_wide_embeddings(E, T, B, din_impl):
    """din_wg_kernel (csrc/din_wg.cu) with E padded to 64: two K blocks per history row, several 64-position
    tiles per row."""
    spec = default_spec("din", emb_dim=E, hist_len=T, n_movies=50_000, n_users=5000)
    W = init_weights(spec, E * 1000 + T)
    feats = synthetic_features(spec, B, seed=T, uniform_history=(T == 200))
    din_impl("tc")
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        p_rt, z_rt = m.predict_with_logits(feats)
        p_rt2 = m.predict(feats)
    assert np.array_equal(p_rt, p_rt2)                       # deterministic
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z_rt - zo).max() <= 5e-4, "logit err %g" % np.abs(z_rt - zo).max()
    assert np.abs(p_rt - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p_rt - po).max()
    din_impl("cudacore")
    with _model(spec, W) as m:
        assert m.kernel_name == "din_kernel"
        p_cc = m.predict(feats)
    assert np.abs(p_cc - p_rt).max() <= 2 * PROB_ATOL


def test_din_row_tile_kernel_wide_row_independence(din_impl):
    din_impl("tc")
    spec = default_spec("din", emb_dim=64, hist_len=200, n_movies=300_000, n_users=5000)
    W = init_weights(spec, 7)
    B = 2 * 148 * 32 + 77
    feats = synthetic_features(spec, B, seed=7, uniform_history=True)
    perm = np.random.default_rng(2).permutation(B)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        p = m.predict(feats)[:, 0]
        pp = m.predict({k: v[perm] for k, v in feats.items()})[:, 0]
        assert np.array_equal(pp, p[perm])                   # bit-exact under row permutation
        lo = m.predict({k: v[:4099] for k, v in feats.items()})[:, 0]
        hi = m.predict({k: v[4099:] for k, v in feats.items()})[:, 0]
        assert np.array_equal(np.concatenate([lo, hi]), p)   # sharding invariant


@pytest.mark.parametrize("sm_cap", [0, 7])
def test_din_tensor_core_row_independence(sm_cap, din_impl):
    din_impl("tc")
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 3)
    B = 8192 + 5
    feats = synthetic_features(spec, B, seed=3)
    perm = np.random.default_rng(1).permutation(B)
    with _model(spec, W) as m:
        m.set_sm_limit(sm_cap)
        p = m.predict(feats)[:, 0]
        pp = m.predict({k: v[perm] for k, v in feats.items()})[:, 0]
        assert np.array_equal(pp, p[perm])                   # bit-exact under row permutation
        assert m.kernel_name == "din_wg_kernel"
        lo = m.predict({k: v[:4099] for k, v in feats.items()})[:, 0]
        hi = m.predict({k: v[4099:] for k, v in feats.items()})[:, 0]
        assert np.array_equal(np.concatenate([lo, hi]), p)   # sharding invariant


@pytest.mark.parametrize("sm_cap", [0, 7])
def test_din_tensor_core_large_magnitudes(sm_cap, din_impl):
    """Trained-scale weights: embeddings O(0.5), logits up to ~10 - the bf16x3 split must hold
    the 1e-4 target with margin where plain TF32/bf16 would not."""
    din_impl("tc")
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 5)
    W["embedding"] = (W["embedding"] * 10).astype(np.float32)
    W["dense_2/kernel"] = (W["dense_2/kernel"] * 4).astype(np.float32)
    feats = synthetic_features(spec, 2048, seed=5)
    with _model(spec, W) as m:
        m.set_sm_limit(sm_cap)
        p, z = m.predict_with_logits(feats)
    po, zo = O.forward(spec, W, feats)
    assert np.abs(zo).max() > 2.0
    assert np.abs(p - po).max() <= 1e-4, np.abs(p - po).max()     # the north_star target
    assert np.abs(z - zo).max() <= 1e-3 * max(1.0, np.abs(zo).max())


def test_predict_batches_packed_and_unpacked_agree():
    """`srs_predict_host_batches`: packed arenas (one H2D copy) and scattered arrays (one copy
    per array) give the same scores as the single-batch call; Keras-style batched predict."""
    spec = default_spec("din", emb_dim=32, hist_len=20, n_movies=3000, n_users=2000)
    W = init_weights(spec, 12)
    feats = synthetic_features(spec, 5000, seed=12)
    with _model(spec, W) as m:
        ref = m.predict(feats)[:, 0]
        encs, outs = [], []
        for lo in range(0, 5000, 700):
            sub = {k: v[lo:lo + 700] for k, v in feats.items()}
            encs.append(encode_batch(spec, sub))                    # packed arena
            outs.append(np.empty(encs[-1].B, np.float32))
        m.predict_batches(encs, outs)
        assert np.array_equal(np.concatenate(outs), ref)
        scattered = []
        for e in encs:                                              # break the adjacency
            scattered.append(type(e)(e.B, e.movie_id.copy(), e.user_id.copy(), e.hist.copy(),
                                     e.movie_genre.copy(), e.user_genre.copy(), e.numerics.copy()))
        outs2 = [np.empty(e.B, np.float32) for e in scattered]
        m.predict_batches(scattered, outs2)
        assert np.array_equal(np.concatenate(outs2), ref)
        assert np.array_equal(m.predict(feats, batch_size=12 * 50)[:, 0], ref)


# ---- EmbeddingMLP / Wide&Deep tensor-core kernel (csrc/embmlp_tc.cu) ----------------------
@pytest.mark.parametrize("model", ["embeddingmlp", "widendeep"])
@pytest.mark.parametrize("B", [1, 63, 64, 65, 129, 8192])
def test_embmlp_tensor_core_kernel(model, B, monkeypatch):
    spec = default_spec(model)
    W = init_weights(spec, 31 + B)
    feats = synthetic_features(spec, B, seed=B)
    monkeypatch.setenv("SRS_EMBMLP_IMPL", "tc")
    with _model(spec, W) as m:
        assert m.kernel_name.startswith("embmlp_tc_kernel")
        p_tc, z_tc = m.predict_with_logits(feats)
        assert np.array_equal(m.predict(feats), p_tc)
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z_tc - zo).max() <= LOGIT_ATOL, "logit err %g" % np.abs(z_tc - zo).max()
    assert np.abs(p_tc - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p_tc - po).max()
    monkeypatch.setenv("SRS_EMBMLP_IMPL", "cudacore")
    with _model(spec, W) as m:
        assert m.kernel_name.startswith("embmlp_kernel")
        p_cc = m.predict(feats)
    assert np.abs(p_cc - po).max() <= PROB_ATOL


def test_embmlp_tensor_core_narrow_hidden_and_small_emb(monkeypatch):
    monkeypatch.setenv("SRS_EMBMLP_IMPL", "tc")
    for E, hidden in ((10, (64, 32)), (8, (128, 128)), (12, (100, 77))):
        spec = default_spec("widendeep", emb_dim=E, hidden=hidden, n_movies=2000, n_users=3000)
        W = init_weights(spec, E)
        feats = synthetic_features(spec, 700, seed=E)
        _compare(spec, W, feats)


# ---- DeepFM tensor-core kernel (csrc/deepfm_tc.cu) ---------------------------------------
@pytest.mark.parametrize("E,B", [(16, 4096), (16, 1), (16, 31), (16, 33), (14, 700), (16, 9000)])
def test_deepfm_tensor_core_kernel(E, B, monkeypatch):
    spec = default_spec("deepfm", emb_dim=E, n_movies=27279, n_users=20000)
    W = init_weights(spec, 50 + E + B)
    feats = synthetic_features(spec, B, seed=B + E)
    monkeypatch.setenv("SRS_DEEPFM_IMPL", "tc")
    with _model(spec, W) as m:
        assert m.kernel_name == "deepfm_tc_kernel"
        p_tc, z_tc = m.predict_with_logits(feats)
        assert np.array_equal(m.predict(feats), p_tc)
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z_tc - zo).max() <= LOGIT_ATOL, "logit err %g" % np.abs(z_tc - zo).max()
    assert np.abs(p_tc - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p_tc - po).max()
    monkeypatch.setenv("SRS_DEEPFM_IMPL", "cudacore")
    with _model(spec, W) as m:
        assert m.kernel_name == "deepfm_kernel"
        assert np.abs(m.predict(feats) - po).max() <= PROB_ATOL


# ---- the tensor-core DIN kernel under an SM limit ----------------------------------------------------
# din_wg_kernel walks the batch's 32-row tiles in a grid-stride loop; the SM limit decides how many tiles a
# CTA walks (1 SM: every tile of the batch on one CTA - buffer reuse across tiles, odd last tiles, one-row
# tiles all get exercised).
@pytest.mark.parametrize("E,T,B,sms", [(32, 50, 28, 0), (32, 50, 4096, 0), (32, 50, 4096, 74), (32, 50, 4096, 37),
                                       (32, 50, 1500, 3), (32, 9, 100, 1), (32, 31, 17, 0), (32, 64, 333, 2),
                                       (20, 33, 15, 0), (32, 50, 2 * 148 * 32 + 77, 0), (32, 50, 1, 0),
                                       (32, 50, 223, 1), (24, 17, 2, 0), (32, 50, 9000, 148)])
def test_din_rtp_kernel(E, T, B, sms, din_impl):
    spec = default_spec("din", emb_dim=E, hist_len=T, n_movies=27279, n_users=5000)
    W = init_weights(spec, E * 1000 + T)
    feats = synthetic_features(spec, B, seed=T + B)
    din_impl("tc")
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        if sms:
            m.set_sm_limit(sms)
        p, z = m.predict_with_logits(feats)
        assert np.array_equal(m.predict(feats), p)                 # deterministic
        m.status()                                                 # raises with a diagnosis if a wait timed out
        m.set_sm_limit(5)                                          # results do not depend on the grid
        assert np.array_equal(m.predict(feats), p)
        m.status()
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z - zo).max() <= LOGIT_ATOL, "logit err %g" % np.abs(z - zo).max()
    assert np.abs(p - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p - po).max()


def test_din_rtp_out_of_range_ids_latch_the_error_flag(din_impl):
    from sparrowrecsys_b200._lib import SrsError
    spec = default_spec("din", emb_dim=32, hist_len=50, n_movies=27279, n_users=5000)
    W = init_weights(spec, 1)
    feats = synthetic_features(spec, 300, seed=3)
    din_impl("tc")
    with _model(spec, W) as m:
        d = m.to_device(feats)
        import torch
        d.hist[17, 3] = spec.n_movies + 5                          # device path: no host pre-validation
        out = torch.empty(300, dtype=torch.float32, device="cuda:0")
        m.predict_device(d, out)
        with pytest.raises((SrsError, ValueError)):
            m.status()


@pytest.mark.parametrize("E,T,pos", [(64, 200, 3), (64, 200, 130), (32, 50, 49)])
def test_din_tensor_core_negative_history_id_latches_the_error_flag(E, T, pos, din_impl):
    """-1 is a value a caller can put into a history slot: the tensor-core DIN kernel (the default when E pads
    to 64) range-checks it like every other live id instead of taking it for an empty slot."""
    import torch
    from sparrowrecsys_b200._lib import SrsError
    spec = default_spec("din", emb_dim=E, hist_len=T, n_movies=27279, n_users=5000)
    W = init_weights(spec, 2)
    feats = synthetic_features(spec, 300, seed=4)
    din_impl("tc")
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        d = m.to_device(feats)
        out = torch.empty(300, dtype=torch.float32, device="cuda:0")
        m.predict_device(d, out)
        m.status()                                                 # the valid batch raises nothing
        d.hist[17, pos] = -1                                       # device path: no host pre-validation
        m.predict_device(d, out)
        with pytest.raises((SrsError, ValueError)):
            m.status()
