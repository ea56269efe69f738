"""din_wg_kernel at E <= 32 (csrc/din_wg.cu): the warpgroups of a CTA share a 32-row tile, warpgroup q walking rows
q, q + G, ...; the top-MLP weight image shares shared memory with their history tiles, so the part of it under
the tiles is copied again in every tile.  Checked against the float64 oracle and din_kernel, with the tolerances
of tests/test_gpu_din_wg_pipeline.py (needs a GPU: pytest -m gpu)."""
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


def _check(spec, W, feats, caps=(1, 7, 0)):
    """wgmma kernel against the float64 oracle and din_kernel; scores bit-identical under every grid cap."""
    with _model(spec, W, "tc") as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
        for n in caps:
            m.set_sm_limit(n)
            assert np.array_equal(m.predict(feats), p), n
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z - zo).max() <= LOGIT_ATOL, "logit err %g" % np.abs(z - zo).max()
    assert np.abs(p - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p - po).max()
    with _model(spec, W, "cudacore") as m:
        assert m.kernel_name == "din_kernel"
        p_cc = m.predict(feats)
    assert np.abs(p_cc - p).max() <= 2 * PROB_ATOL
    return p


# B = 32 + r: a full first tile, then a last tile of r rows, so for any warpgroup count every warpgroup gets
# each row count from 0 to its share of a full tile in the last tile
@pytest.mark.parametrize("r", list(range(1, 33)))
def test_last_tile_rows_t50(r):
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 400 + r)
    _check(spec, W, synthetic_features(spec, 32 + r, seed=400 + r), caps=(1, 0))


@pytest.mark.parametrize("r", [1, 3, 4, 5, 7, 8, 9, 13, 31, 32])
def test_last_tile_rows_multi_chunk(r):
    """T = 129: three 64-position items per row, the last one of a single position."""
    spec = default_spec("din", emb_dim=32, hist_len=129, n_movies=27279, n_users=5000)
    W = init_weights(spec, 500 + r)
    _check(spec, W, synthetic_features(spec, 32 + r, seed=500 + r), caps=(1, 0))


def test_one_cta_reloads_the_image_over_many_tiles():
    """B = 4097 under grid caps 1 and 7: one CTA walks 129 (or ~19) tiles, copying the image part under the
    history tiles again in each; the scores stay bit-identical to one tile per CTA."""
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 31)
    _check(spec, W, synthetic_features(spec, 4097, seed=31))


def test_two_streams_under_half_the_sms_match_serial_launches_e32():
    """bench.py's default mode at cfg 3: two launches in flight on two streams, each capped to SMs / 2 CTAs."""
    import torch
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 32)
    B = 4096
    fa, fb = synthetic_features(spec, B, seed=321), synthetic_features(spec, B, seed=322)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
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


def test_packed_w1_tail_alone_over_many_tiles():
    """Only the movie-genre slot (the packed K tail of the W1 image) feeds Dense(128), scaled up, and one CTA
    walks every tile: a tail or a W2 image half read from a stale buffer in a later tile would move the
    logits far outside the tolerance."""
    spec = baseline_spec("cfg3_din")
    E = spec.emb_dim
    W = init_weights(spec, 33)
    g0 = 3 + 2 * E + 2 * E + 1                           # movieGenre1 in Keras's Dense(128) input order
    k1 = np.zeros_like(W["dense/kernel"])
    k1[g0:g0 + E] = 20.0 * W["dense/kernel"][g0:g0 + E]
    W["dense/kernel"] = k1
    feats = synthetic_features(spec, 2048, seed=33)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
        m.set_sm_limit(1)
        p1, z1 = m.predict_with_logits(feats)
    assert np.array_equal(p1, p) and np.array_equal(z1, z)
    po, zo = O.forward(spec, W, feats)
    assert zo.std() > 0.5, zo.std()
    assert np.abs(z - zo).max() <= 1e-5 * max(1.0, np.abs(zo).max()) + LOGIT_ATOL, np.abs(z - zo).max()
    assert np.abs(p - po).max() <= 1e-4, np.abs(p - po).max()
