"""din_wg_kernel as the default DIN kernel at E <= 32 (csrc/din_wg.cu): top MLP on wgmma, vectorised
pooling, grid-stride walk under srs_model_set_sm_limit (needs a GPU: pytest -m gpu)."""
import numpy as np
import pytest

from oracle import ctr_oracle as O
from sparrowrecsys_b200.features import synthetic_features
from sparrowrecsys_b200.spec import baseline_spec, default_spec
from sparrowrecsys_b200.weights import init_weights

pytestmark = pytest.mark.gpu

PROB_ATOL = 2e-5
LOGIT_ATOL = 2e-4


def _model(spec, W, impl=None):
    from sparrowrecsys_b200.model import CTRModel
    return CTRModel(spec, W, device=0, options={"din_impl": impl} if impl else None)


def _n_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _against_oracle_and_cudacore(spec, W, feats, p, z, logit_atol=LOGIT_ATOL, prob_atol=PROB_ATOL):
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z - zo).max() <= logit_atol, "logit err %g" % np.abs(z - zo).max()
    assert np.abs(p - po).max() <= prob_atol, "prob err %g" % np.abs(p - po).max()
    with _model(spec, W, "cudacore") as m:
        assert m.kernel_name == "din_kernel"
        p_cc = m.predict(feats)
    assert np.abs(p_cc - p).max() <= 2 * PROB_ATOL


def test_cfg3_selects_the_wgmma_kernel_by_default():
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 1)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
    with _model(spec, W, "cudacore") as m:
        assert m.kernel_name == "din_kernel"
    short = default_spec("din", emb_dim=32, hist_len=8, n_movies=3000, n_users=500)
    with _model(short, init_weights(short, 1)) as m:
        assert m.kernel_name == "din_kernel"                       # T <= 8 keeps the CUDA-core kernel
    narrow = default_spec("din", emb_dim=16, hist_len=50, n_movies=3000, n_users=500)
    with _model(narrow, init_weights(narrow, 1)) as m:
        assert m.kernel_name == "din_kernel"                       # E <= 16: the only kernel


@pytest.mark.parametrize("B", [4096, 4097])
def test_scores_do_not_depend_on_the_grid(B):
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 3)
    feats = synthetic_features(spec, B, seed=B)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        ref = m.predict(feats)
        for n in (1, 7, _n_sms() // 2, 0):
            m.set_sm_limit(n)
            assert np.array_equal(m.predict(feats), ref), n


def test_two_streams_under_half_the_sms_match_serial_launches():
    """bench.py's default mode: two launches in flight on two streams, each capped to SMs / 2 CTAs."""
    import torch
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 4)
    B = 4096
    fa, fb = synthetic_features(spec, B, seed=41), synthetic_features(spec, B, seed=42)
    with _model(spec, W) as m:
        ra, rb = m.predict(fa)[:, 0], m.predict(fb)[:, 0]
        da, db = m.to_device(fa), m.to_device(fb)
        m.set_sm_limit(_n_sms() // 2)
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        outs = [torch.empty(B, dtype=torch.float32, device="cuda:0") for _ in range(8)]
        for s in (s1, s2):
            s.wait_stream(torch.cuda.current_stream())
        for i in range(8):
            m.predict_device(da if i % 2 == 0 else db, outs[i], stream=s1 if i % 2 == 0 else s2)
        for s in (s1, s2):
            torch.cuda.current_stream().wait_stream(s)
        m.status()
        for i in range(8):
            assert np.array_equal(outs[i].cpu().numpy(), ra if i % 2 == 0 else rb), i


@pytest.mark.parametrize("T", [1, 9, 63, 64, 65, 129])
@pytest.mark.parametrize("B", [1, 31, 33, 4097])
def test_ring_and_tile_edges(T, B):
    spec = default_spec("din", emb_dim=32, hist_len=T, n_movies=27279, n_users=5000)
    W = init_weights(spec, 100 + T)
    feats = synthetic_features(spec, B, seed=T * 7 + B)
    with _model(spec, W, "tc") as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
        m.set_sm_limit(1)                                          # one CTA walks every tile of the batch
        assert np.array_equal(m.predict(feats), p)
    _against_oracle_and_cudacore(spec, W, feats, p, z)


def test_top_mlp_hidden_widths_below_the_padding():
    spec = default_spec("din", emb_dim=32, hist_len=50, hidden=(100, 40), n_movies=27279, n_users=5000)
    W = init_weights(spec, 11)
    feats = synthetic_features(spec, 777, seed=11)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
    _against_oracle_and_cudacore(spec, W, feats, p, z)


def test_top_mlp_numerics_scaled_up():
    """The 7 numerics stay out of the MMAs (fp32 in the layer-1 epilogue).  x100 numerics make the hidden
    activations ~100x larger, so the bf16x3 products downstream carry ~100x the absolute error: held to the
    north-star 1e-4 on probabilities and 1e-5 relative on logits, far below what rounding a numeric's
    contribution to bf16 (2^-9 relative) would leave."""
    from sparrowrecsys_b200.spec import NUMERIC_KEYS
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 12)
    feats = synthetic_features(spec, 1000, seed=12)
    for k in NUMERIC_KEYS:
        feats[k] = (np.asarray(feats[k], np.float32) * 100).astype(np.float32)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z - zo).max() <= 1e-5 * max(1.0, np.abs(zo).max()) + LOGIT_ATOL
    assert np.abs(p - po).max() <= 1e-4, np.abs(p - po).max()


def test_top_mlp_trained_magnitudes():
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 13)
    W["embedding"] = (W["embedding"] * 10).astype(np.float32)
    W["dense/kernel"] = (W["dense/kernel"] * 3).astype(np.float32)
    W["dense_2/kernel"] = (W["dense_2/kernel"] * 4).astype(np.float32)
    feats = synthetic_features(spec, 2048, seed=13)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
    po, zo = O.forward(spec, W, feats)
    assert np.abs(zo).max() > 2.0
    assert np.abs(p - po).max() <= 1e-4, np.abs(p - po).max()
    assert np.abs(z - zo).max() <= 1e-3 * max(1.0, np.abs(zo).max())


@pytest.mark.parametrize("what", ["candidate", "history"])
def test_range_errors_latch_under_the_default(what):
    import torch
    from sparrowrecsys_b200._lib import SrsError
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 14)
    feats = synthetic_features(spec, 300, seed=14)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        d = m.to_device(feats)
        out = torch.empty(300, dtype=torch.float32, device="cuda:0")
        m.predict_device(d, out)
        m.status()
        if what == "candidate":
            d.movie_id[200] = spec.n_movies
        else:
            d.hist[17, 49] = -1
        m.predict_device(d, out)
        with pytest.raises((SrsError, ValueError)):
            m.status()
