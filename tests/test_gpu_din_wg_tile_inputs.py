"""din_wg_kernel's tile inputs under a grid cap (csrc/din_wg.cu): a CTA that walks several tiles requests the ids of
each tile at its start, copies the side features asynchronously and (E <= 32) lets each warpgroup copy
the candidate rows of its own rows.  An out-of-range id in the tile a CTA reaches second still latches the error
word, and every other row scores exactly as in the uncapped launch (needs a GPU: pytest -m gpu)."""
import numpy as np
import pytest

from sparrowrecsys_b200.features import encode_batch, synthetic_features
from sparrowrecsys_b200.spec import baseline_spec, default_spec
from sparrowrecsys_b200.weights import init_weights

pytestmark = pytest.mark.gpu

CAP = 3                                   # CTAs per launch: CTA c walks tiles c, c + 3, c + 6


@pytest.mark.parametrize("bad", ["user_id", "user_genre", "hist"])
@pytest.mark.parametrize("E,T", [(32, 50), (64, 200)], ids=["ep32", "ep64"])
def test_a_bad_id_in_a_ctas_second_tile_latches_and_leaves_the_other_rows(E, T, bad):
    """One out-of-range id per launch, so that each range check (user id, genre, history id) is held on its own."""
    import torch
    from sparrowrecsys_b200.model import CTRModel
    spec = baseline_spec("cfg3_din") if E == 32 else \
        default_spec("din", emb_dim=E, hist_len=T, n_movies=27279, n_users=5000)
    W = init_weights(spec, 61)
    B = 32 * 2 * CAP + 5                  # 7 tiles: the last one partial, walked third by CTA 0
    feats = synthetic_features(spec, B, seed=61)
    tile = CAP + 1                        # CTA 1's second tile
    row = 32 * tile + {"user_id": 1, "user_genre": 6, "hist": 11}[bad]
    with CTRModel(spec, W, device=0, options={"din_impl": "tc"}) as m:
        assert m.kernel_name == "din_wg_kernel"
        ref = m.predict(feats)[:, 0]
        m.status()                        # the valid batch latches nothing
        enc = encode_batch(spec, feats)
        col = np.array(getattr(enc, bad), copy=True)
        if bad == "user_id":
            col[row] = spec.n_users + 3
        elif bad == "user_genre":
            col[row, 0] = spec.n_genres + 2
        else:
            col[row, 3] = spec.n_movies + 7
        setattr(enc, bad, col)
        d = m.to_device(enc)
        got = {}
        for cap in (0, CAP):
            m.set_sm_limit(cap)
            out = torch.empty(B, dtype=torch.float32, device="cuda:0")
            m.predict_device(d, out)
            with pytest.raises(ValueError):
                m.status()
            m.status()                    # cleared by the report
            got[cap] = out.cpu().numpy()
    assert np.array_equal(got[CAP], got[0])
    keep = np.arange(B) != row
    assert np.array_equal(got[CAP][keep], ref[keep])
