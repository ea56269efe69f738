"""din_wg_kernel's row walk (csrc/din_wg.cu): three warpgroups share a 32-row tile, each walking every third
row in (row, 64-position chunk) items, so a warpgroup may get 0, 1, 2 or more rows of a batch's last tile and a
row may span several items; and the packed W1 tail of the top-MLP image (needs a GPU: pytest -m gpu)."""
import numpy as np
import pytest

from oracle import ctr_oracle as O
from sparrowrecsys_b200.features import synthetic_features
from sparrowrecsys_b200.spec import baseline_spec, default_spec
from sparrowrecsys_b200.weights import init_weights

pytestmark = pytest.mark.gpu

PROB_ATOL = 2e-5                 # as tests/test_gpu_din_pipeline.py
LOGIT_ATOL = 2e-4


def _model(spec, W, impl=None):
    from sparrowrecsys_b200.model import CTRModel
    return CTRModel(spec, W, device=0, options={"din_impl": impl} if impl else None)


def _n_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check(spec, W, feats):
    """wgmma kernel against the float64 oracle and din_kernel; scores bit-identical under every grid cap."""
    with _model(spec, W, "tc") as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
        for n in (1, 7, 0):
            m.set_sm_limit(n)
            assert np.array_equal(m.predict(feats), p), n
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z - zo).max() <= LOGIT_ATOL, "logit err %g" % np.abs(z - zo).max()
    assert np.abs(p - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p - po).max()
    with _model(spec, W, "cudacore") as m:
        assert m.kernel_name == "din_kernel"
        p_cc = m.predict(feats)
    assert np.abs(p_cc - p).max() <= 2 * PROB_ATOL


# B mod 32 sets the rows of the last 32-row tile, dealt to the three warpgroups in turn: 0, 1 or 2 rows each for
# B mod 32 in 1 .. 5, 10 or 11 for B = 63, a one-row last tile for B = 33, 65, 4097
ITEM_BATCHES = [1, 2, 3, 4, 5, 33, 63, 65, 4097]


@pytest.mark.parametrize("T", [9, 50, 64, 65, 128, 129])
@pytest.mark.parametrize("B", ITEM_BATCHES)
def test_item_count_edges_e32(B, T):
    spec = default_spec("din", emb_dim=32, hist_len=T, n_movies=27279, n_users=5000)
    W = init_weights(spec, 200 + T)
    _check(spec, W, synthetic_features(spec, B, seed=3 * T + B))


@pytest.mark.parametrize("E", [48, 64])
@pytest.mark.parametrize("T", [9, 65, 200])
@pytest.mark.parametrize("B", ITEM_BATCHES)
def test_item_count_edges_e64(B, T, E):
    spec = default_spec("din", emb_dim=E, hist_len=T, n_movies=27279, n_users=5000)
    W = init_weights(spec, 300 + T + E)
    _check(spec, W, synthetic_features(spec, B, seed=5 * T + B + E))


def test_permuted_rows_give_permuted_scores():
    """A row that read another warpgroup's W_r, gate weights or parts would change with the permutation."""
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 21)
    B = 4096
    feats = synthetic_features(spec, B, seed=21)
    perm = np.random.default_rng(21).permutation(B)
    permuted = {k: np.asarray(v)[perm] for k, v in feats.items()}
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        ref = m.predict(feats)
        got = m.predict(permuted)
    assert np.array_equal(got, ref[perm])


def test_two_streams_under_half_the_sms_match_serial_launches_e64():
    """bench.py's default mode at E = 64: two launches in flight on two streams, each capped to SMs / 2 CTAs."""
    import torch
    spec = default_spec("din", emb_dim=64, hist_len=200, n_movies=27279, n_users=5000)
    W = init_weights(spec, 22)
    B = 4096
    fa, fb = synthetic_features(spec, B, seed=221), synthetic_features(spec, B, seed=222)
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


def test_packed_w1_tail_alone():
    """Only the movie-genre slot - tile columns 128..159, the K tail packed as [hi | lo] in one block of the
    W1 image - feeds Dense(128), scaled up.  A tail read with the wrong swizzle or the wrong half moves the
    logits by about their spread; a lost lo half by ~2^-9 of it.  Both are far outside the tolerance."""
    spec = baseline_spec("cfg3_din")
    E = spec.emb_dim
    W = init_weights(spec, 23)
    # Dense(128) input in Keras order: [userAvgRating, userGenre1 (E), userId (E), userRatingCount,
    # userRatingStddev | pooled (E) | candidate (E) | movieAvgRating, movieGenre1 (E), ...]
    g0 = 3 + 2 * E + 2 * E + 1
    k1 = np.zeros_like(W["dense/kernel"])
    k1[g0:g0 + E] = 20.0 * W["dense/kernel"][g0:g0 + E]
    W["dense/kernel"] = k1
    feats = synthetic_features(spec, 2048, seed=23)
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
    po, zo = O.forward(spec, W, feats)
    assert zo.std() > 0.5, zo.std()                       # the tail alone moves the logits
    assert np.abs(z - zo).max() <= 1e-5 * max(1.0, np.abs(zo).max()) + LOGIT_ATOL, np.abs(z - zo).max()
    assert np.abs(p - po).max() <= 1e-4, np.abs(p - po).max()
