"""DIEN's second output (the auxiliary-loss head, DIEN.py:261-296) and its Keras evaluate.

The float64 restatement of the head lives here, beside the tests that use it: it reuses
`oracle.ctr_oracle`'s pieces (dense, sigmoid, numeric) and restates `dien_forward`'s GRU loop to get the
per-position outputs g_t that `dien_forward` does not return.
"""
import os

import numpy as np
import pytest

from oracle import ctr_oracle as O
from oracle import keras_eval as K

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- oracle ------------------------------------------------------------------------------------------------
def neg_keys(T):
    return ["negtive_userRatedMovie%d" % k for k in range(2, T + 1)]


def gru_outputs(spec, W, feats):
    """g_1..g_T of DIEN.py:169 in float64 (the GRU of oracle/ctr_oracle.py::dien_forward: Keras z | r | h,
    reset_after, a masked position carries state and output), the embedding table and the history ids."""
    E, T = spec.emb_dim, spec.hist_len
    hist_f = np.concatenate([O.numeric(feats, k, np.float32) for k in O.din_history_keys(T)], axis=1)
    hist = hist_f.astype(np.int32)
    mask = hist_f != 0
    tab = W["embedding"].astype(np.float64)
    X = tab[hist]
    Kk, U = W["gru/kernel"].astype(np.float64), W["gru_recurrent/kernel"].astype(np.float64)
    bx, bh = W["gru/bias"].astype(np.float64)
    h = np.zeros((hist.shape[0], E))
    G = np.zeros((hist.shape[0], T, E))
    for t in range(T):
        mx = X[:, t] @ Kk + bx
        mh = h @ U + bh
        z = O.sigmoid(mx[:, :E] + mh[:, :E])
        r = O.sigmoid(mx[:, E:2 * E] + mh[:, E:2 * E])
        hh = np.tanh(mx[:, 2 * E:] + r * mh[:, 2 * E:])
        h = np.where(mask[:, t, None], z * h + (1 - z) * hh, h)
        G[:, t] = h
    return G, tab, hist


def neg_ids(spec, feats):
    T = spec.hist_len
    if T == 1:
        return np.zeros((len(feats["movieId"]), 0), np.int32)
    neg = np.concatenate([O.numeric(feats, k, np.float32) for k in neg_keys(T)], axis=1).astype(np.int32)
    if neg.size and (neg.min() < 0 or neg.max() >= spec.n_movies):
        raise ValueError("negative movie id out of range")
    return neg


def aux_oracle(spec, W, feats, defect=None):
    """aux_row = sum_{t=1}^{T-1} pos_t + neg_t (DIEN.py:276-285): Dense32(sigmoid) then Dense1(sigmoid) over
    [g_t | e(h_{t+1})] and [g_t | e(n_{t+1})], 1-based; no mask (the slices drop it).  `defect` "last" (a mutant
    for the tests) leaves the sum's last step t = T - 1 out."""
    G, tab, hist = gru_outputs(spec, W, feats)
    neg = neg_ids(spec, feats)
    W64 = {k: v.astype(np.float64) for k, v in W.items() if k.startswith("aux_")}

    def head(side, g, e):
        x = np.concatenate([g, e], axis=1)                 # hidden state first (DIEN.py:278,282)
        return O.dense(O.dense(x, W64, "aux_%s_dense" % side, "sigmoid"), W64, "aux_%s_out" % side, "sigmoid")[:, 0]
    aux = np.zeros(hist.shape[0])
    for t in range(1, spec.hist_len - (defect == "last")):  # 0-based t: g_t = G[t-1], next item = position t
        aux += head("pos", G[:, t - 1], tab[hist[:, t]]) + head("neg", G[:, t - 1], tab[neg[:, t - 1]])
    return aux


def aux_literal(spec, W, feats):
    """The same head as a literal per-row, per-position loop (1-based t as in DIEN.py)."""
    G, tab, hist = gru_outputs(spec, W, feats)
    neg = neg_ids(spec, feats)
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    out = np.zeros(hist.shape[0])
    for i in range(hist.shape[0]):
        for t in range(1, spec.hist_len):                  # 1-based t = 1..T-1
            g = G[i, t - 1]
            for side, e in (("pos", tab[hist[i, t]]), ("neg", tab[neg[i, t - 1]])):
                x = np.concatenate([g, e])
                Wd, bd = W["aux_%s_dense/kernel" % side].astype(np.float64), W["aux_%s_dense/bias" % side]
                Wo, bo = W["aux_%s_out/kernel" % side].astype(np.float64), W["aux_%s_out/bias" % side]
                hid = np.array([sig(sum(x[k] * Wd[k, j] for k in range(x.shape[0])) + bd[j]) for j in range(32)])
                out[i] += sig(float(hid @ Wo[:, 0]) + float(bo[0]))
    return out


def final_loss_oracle(logits, labels, aux, batch_size=None):
    """DIEN.py:287 per Keras batch: bce_i - 0.5 * mean_{j in batch} aux_j, bce on the logit path (float32 per
    row, keras_eval.logit_bce_f32), the rest in float64."""
    n = len(aux)
    step = n if not batch_size else batch_size
    bce = K.logit_bce_f32(logits, labels).astype(np.float64)
    out = np.empty(n)
    for lo in range(0, n, step):
        out[lo:lo + step] = bce[lo:lo + step] - 0.5 * np.mean(np.asarray(aux[lo:lo + step], np.float64))
    return out


def auc_value_oracle(probs, labels, batch_size):
    """add_metric(auc.result(), aggregation="mean"): the mean over batches k of the ROC AUC of batches 0..k,
    each from exact counts in double."""
    n = len(probs)
    aucs = [K.roc_auc_from_counts(*K.confusion_counts(probs[:hi], labels[:hi]))
            for hi in [min(n, lo + batch_size) for lo in range(0, n, batch_size)]]
    return float(np.mean(aucs))


def aux_weights(spec, seed):
    """`init_aux_weights` with non-zero biases, so that every tensor of the group shows in the output."""
    from sparrowrecsys_b200.weights import init_aux_weights
    W = init_aux_weights(spec, seed)
    rng = np.random.default_rng(seed + 100)
    for k in W:
        if k.endswith("/bias"):
            W[k] = rng.uniform(-0.3, 0.3, size=W[k].shape).astype(np.float32)
    return W


def with_negatives(spec, feats, seed):
    from sparrowrecsys_b200.features import negative_history
    f = dict(feats)
    f.update(negative_history(feats, spec.hist_len, seed, n_movies=spec.n_movies))
    rng = np.random.default_rng(seed)
    f["label"] = (rng.random(len(feats["movieId"])) < 0.4).astype(np.int32)
    return f


# ---- CPU ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [1, 2, 5, 12])
def test_oracle_head_matches_a_literal_loop(T):
    from sparrowrecsys_b200.features import synthetic_features
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    spec = default_spec("dien", hist_len=T, n_movies=500, n_users=300)
    W = {**init_weights(spec, 3), **aux_weights(spec, 3)}
    feats = with_negatives(spec, synthetic_features(spec, 7, seed=T), seed=T)
    got, want = aux_oracle(spec, W, feats), aux_literal(spec, W, feats)
    if T == 1:
        assert np.array_equal(got, np.zeros(7))
    assert np.allclose(got, want, rtol=0, atol=1e-6)
    assert np.all(got > 0) or T == 1


def test_final_loss_of_a_hand_built_batch():
    logits = np.array([0.5, -1.0, 2.0], np.float32)
    labels = np.array([1, 0, 0], np.int32)
    aux = np.array([1.2, 0.6, 3.0])
    bce = [np.log1p(np.exp(-0.5)), np.log1p(np.exp(-1.0)), 2.0 + np.log1p(np.exp(-2.0))]
    want = np.array(bce) - 0.5 * (1.2 + 0.6 + 3.0) / 3
    assert np.allclose(final_loss_oracle(logits, labels, aux), want, atol=1e-6)
    # batches [0, 1] and [2]: each row subtracts half its own batch's mean
    split = np.array([bce[0] - 0.5 * 0.9, bce[1] - 0.5 * 0.9, bce[2] - 0.5 * 3.0])
    assert np.allclose(final_loss_oracle(logits, labels, aux, batch_size=2), split, atol=1e-6)


def test_auc_value_of_two_hand_built_batches():
    p = np.array([0.9, 0.2, 0.6, 0.4, 0.7, 0.1], np.float32)
    y = np.array([1, 0, 0, 1, 1, 0])
    a1 = K.roc_auc_from_counts(*K.confusion_counts(p[:3], y[:3]))
    a2 = K.roc_auc_from_counts(*K.confusion_counts(p, y))
    assert a1 == 1.0                                        # batch 0 alone is separable
    assert abs(a2 - 8 / 9) < 0.02                           # 200 thresholds around the rank AUC 8/9
    assert auc_value_oracle(p, y, 3) == pytest.approx((a1 + a2) / 2, abs=1e-15)


def test_negative_sampler():
    import random
    from sparrowrecsys_b200.features import negative_history
    hist = np.random.default_rng(0).integers(0, 1001, size=(50, 4)).astype(np.int32)
    feats = {"userRatedMovie%d" % (k + 2): hist[:, k] for k in range(4)}
    feats["userRatedMovie3"] = feats["userRatedMovie3"].astype(np.float64)
    feats["userRatedMovie3"][5] = np.nan                    # fillna(0)
    a = negative_history(feats, 5, seed=2021)
    assert list(a) == neg_keys(5)
    for k in range(2, 6):
        pos = np.nan_to_num(np.asarray(feats["userRatedMovie%d" % k], np.float64)).astype(int)
        assert np.all(a["negtive_userRatedMovie%d" % k] != pos)
        assert a["negtive_userRatedMovie%d" % k].min() >= 0 and a["negtive_userRatedMovie%d" % k].max() <= 1000
    b = negative_history(feats, 5, seed=2021)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    assert not np.array_equal(a["negtive_userRatedMovie2"], negative_history(feats, 5, seed=2020)["negtive_userRatedMovie2"])
    # column-major: re-seed, skip the draws of columns 2 and 3, then column 4 comes out the same
    rng = random.Random(2021)
    for _ in range(2 * 50):
        rng.sample(range(1000), 1)
    col4 = [rng.sample(sorted(set(range(1001)) - {int(x)}), 1)[0] for x in hist[:, 2]]
    assert np.array_equal(a["negtive_userRatedMovie4"], col4)


def test_existing_dien_inventory_is_unchanged():
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import (aux_weight_shapes, check_weights, has_aux_weights, init_aux_weights,
                                            init_weights, weight_shapes)
    spec = default_spec("dien")
    names = [n for n, _ in weight_shapes(spec)]
    assert not any(n.startswith("aux_") for n in names)
    W0 = init_weights(spec, 7)
    Wa = init_aux_weights(spec, 7)
    assert [n for n, _ in aux_weight_shapes(spec)] == list(Wa)
    assert dict(aux_weight_shapes(spec))["aux_pos_dense/kernel"] == (2 * spec.emb_dim, 32)
    W1 = init_weights(spec, 7)
    assert list(W0) == list(W1) and all(W0[k].tobytes() == W1[k].tobytes() for k in W0)
    check_weights(spec, {**W0, **Wa})
    assert has_aux_weights(spec, {**W0, **Wa}) and not has_aux_weights(spec, W0)
    with pytest.raises(KeyError):
        has_aux_weights(spec, {**W0, "aux_neg_out/bias": Wa["aux_neg_out/bias"]})
    with pytest.raises(ValueError):
        aux_weight_shapes(default_spec("din"))


def test_dien_evaluate_still_raises():
    import tfrecmodel.dien as D
    with pytest.raises(NotImplementedError, match="auxiliary"):
        D.evaluate({})


# ---- GPU ---------------------------------------------------------------------------------------------------
def _dien(E, T, seed=0, aux=True):
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    spec = default_spec("dien", emb_dim=E, hist_len=T, n_movies=3000, n_users=4000)
    W = init_weights(spec, seed)
    if aux:
        W.update(aux_weights(spec, seed))
    return CTRModel(spec, W), spec, W


@pytest.mark.gpu
@pytest.mark.parametrize("E", [10, 16, 32])
@pytest.mark.parametrize("T", [1, 2, 5, 50])
def test_outputs_against_the_oracle(E, T):
    from sparrowrecsys_b200.features import synthetic_features
    m, spec, W = _dien(E, T, seed=E + T)
    with m:
        for B in (1, 31, 33, 4097):
            feats = with_negatives(spec, synthetic_features(spec, B, seed=B), seed=B)
            p_ref, z_ref = m.predict_with_logits(feats)
            aux_want = aux_oracle(spec, W, feats)
            for bs in (None, 12):
                y, fl = m.dien_outputs(feats, batch_size=bs)
                assert np.array_equal(y, p_ref), (B, bs)
                want = final_loss_oracle(z_ref[:, 0], feats["label"], aux_want, bs)
                assert np.abs(fl - want).max() <= 1e-5, (B, bs, np.abs(fl - want).max())
            # the device entry point: aux itself, and bits equal to the host path as one batch
            import torch
            dev = m.to_device(feats)
            neg = torch.from_numpy(np.ascontiguousarray(neg_ids(spec, feats))).cuda()
            lab = torch.from_numpy(feats["label"]).cuda()
            out = [torch.empty(B, dtype=torch.float32, device="cuda") for _ in range(4)]
            _dien_device(m, dev, neg, max(T - 1, 0), lab, *out)
            m.status()
            probs, logits, aux, fl_dev = (t.cpu().numpy() for t in out)
            assert np.array_equal(probs, p_ref[:, 0]) and np.array_equal(logits, z_ref[:, 0])
            assert np.allclose(aux, aux_want, rtol=1e-5, atol=1e-6), np.abs(aux - aux_want).max()
            assert np.array_equal(fl_dev, m.dien_outputs(feats)[1])


def _dien_device(m, dev, neg, stride, lab, probs, logits, aux, final_loss):
    import ctypes as C
    import torch
    from sparrowrecsys_b200 import _lib
    b = dev.struct()
    _lib.check(m._lib.srs_dien_outputs_device(
        m._h, C.byref(b), neg.data_ptr() if neg.numel() else None, stride, lab.data_ptr(), probs.data_ptr(),
        logits.data_ptr(), aux.data_ptr(), final_loss.data_ptr(), torch.cuda.current_stream().cuda_stream))


def _test_rows():
    from sparrowrecsys_b200.features import negative_history
    z = np.load(os.path.join(GOLDEN, "dien_testset.npz"))
    feats = {k: z[k] for k in z.files}
    feats.update(negative_history(feats, 5, seed=2021))    # DIEN.py:50
    return feats


@pytest.mark.gpu
def test_evaluate_on_the_test_samples():
    from sparrowrecsys_b200.model import CTRModel, Metrics
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    import torch
    spec = default_spec("dien")
    W = {**init_weights(spec, 5), **aux_weights(spec, 5)}
    feats = _test_rows()
    lab = feats["label"]
    with CTRModel(spec, W) as m:
        r = m.dien_evaluate(feats, batch_size=12)
        p, z = m.predict_with_logits(feats)
        y, fl = m.dien_outputs(feats, batch_size=12)
        assert np.array_equal(y, p)
        aux = aux_oracle(spec, W, feats)
        want_loss = float(np.mean(final_loss_oracle(z[:, 0], lab, aux, 12)))
        assert r["loss"] == pytest.approx(want_loss, rel=1e-6)
        assert r["loss"] == pytest.approx(float(np.sum(fl.astype(np.float64)) / len(fl)), rel=1e-12)
        with Metrics() as mt:
            mt.update_device(torch.from_numpy(p[:, 0]).cuda(), torch.from_numpy(z[:, 0]).cuda(),
                             torch.from_numpy(lab).cuda())
            assert r["auc"] == mt.result()["roc_auc"]
        assert abs(r["auc_value"] - auc_value_oracle(p[:, 0], lab, 12)) <= 1e-12
        # the same bits again, and at SM limits 0 and 8
        for limit in (0, 8, 0):
            m.set_sm_limit(limit)
            assert m.dien_evaluate(feats, batch_size=12) == r
            y2, fl2 = m.dien_outputs(feats, batch_size=12)
            assert np.array_equal(y2, y) and np.array_equal(fl2, fl)
        one = m.dien_evaluate(feats)                         # batch_size None: one batch
        assert one["auc"] == r["auc"] and one["auc_value"] == pytest.approx(r["auc"], abs=1e-15)


@pytest.mark.gpu
def test_ragged_last_batch_and_errors_leave_the_model_clean():
    from sparrowrecsys_b200.features import synthetic_features
    m, spec, W = _dien(10, 5, seed=3)
    with m:
        feats = with_negatives(spec, synthetic_features(spec, 100, seed=9), seed=9)
        p_ref, z_ref = m.predict_with_logits(feats)
        aux = aux_oracle(spec, W, feats)
        y, fl = m.dien_outputs(feats, batch_size=12)          # 8 full batches and one of 4
        assert np.abs(fl - final_loss_oracle(z_ref[:, 0], feats["label"], aux, 12)).max() <= 1e-5
        r = m.dien_evaluate(feats, batch_size=12)
        assert abs(r["auc_value"] - auc_value_oracle(p_ref[:, 0], feats["label"], 12)) <= 1e-12
        bad = dict(feats, negtive_userRatedMovie3=feats["negtive_userRatedMovie3"].copy())
        bad["negtive_userRatedMovie3"][40] = spec.n_movies
        for call in (m.dien_outputs, m.dien_evaluate):
            with pytest.raises(ValueError):
                call(bad, batch_size=12)
        with pytest.raises(ValueError):
            m.dien_outputs(dict(feats, label=np.full(100, 2)), batch_size=12)
        with pytest.raises(KeyError):
            m.dien_outputs({k: v for k, v in feats.items() if k != "negtive_userRatedMovie5"})
        with pytest.raises(KeyError):
            m.dien_evaluate({k: v for k, v in feats.items() if k != "label"})
        # an out-of-range negative id that reaches the kernel: SRS_ERR_RANGE, then every call is clean
        import torch
        dev = m.to_device(feats)
        neg = neg_ids(spec, feats)
        neg[7, 2] = spec.n_movies + 5
        neg = torch.from_numpy(np.ascontiguousarray(neg)).cuda()
        out = [torch.empty(100, dtype=torch.float32, device="cuda") for _ in range(4)]
        _dien_device(m, dev, neg, 4, torch.from_numpy(feats["label"]).cuda(), *out)
        with pytest.raises(ValueError):
            m.status()
        m.status()
        y2, fl2 = m.dien_outputs(feats, batch_size=12)
        assert np.array_equal(y2, y) and np.array_equal(fl2, fl)
        assert m.dien_evaluate(feats, batch_size=12) == r
        assert np.array_equal(m.predict(feats), p_ref)


@pytest.mark.gpu
def test_model_without_the_group():
    from sparrowrecsys_b200.features import synthetic_features
    from sparrowrecsys_b200.model import CTRModel
    m_aux, spec, W = _dien(16, 5, seed=4)
    with m_aux, CTRModel(spec, {k: v for k, v in W.items() if not k.startswith("aux_")}) as m:
        feats = with_negatives(spec, synthetic_features(spec, 50, seed=4), seed=4)
        assert np.array_equal(m.predict(feats), m_aux.predict(feats))
        with pytest.raises(ValueError, match="auxiliary"):
            m.dien_outputs(feats)
        with pytest.raises(ValueError, match="auxiliary"):
            m.dien_evaluate(feats)
        with pytest.raises(ValueError, match="DIEN"):
            m_aux.evaluate(feats)
    from sparrowrecsys_b200.spec import default_spec
    from sparrowrecsys_b200.weights import init_weights
    din = default_spec("din", n_movies=3000, n_users=4000)
    with CTRModel(din, init_weights(din, 0)) as m:
        with pytest.raises(ValueError, match="not DIEN"):
            m.dien_evaluate(with_negatives(din, synthetic_features(din, 20, seed=1), seed=1))


@pytest.mark.gpu
def test_tfrecmodel_surface():
    import tfrecmodel.dien as D
    feats = _test_rows()
    feats = {k: v[:240] for k, v in feats.items()}
    D.load(seed=1)
    y, fl = D.predict_outputs(feats, batch_size=12)
    assert np.array_equal(y, D.predict(feats, batch_size=12)) and fl.shape == (240,)
    r = D.evaluate_outputs(feats, batch_size=12)
    assert set(r) == {"loss", "auc", "auc_value"}
    assert r["loss"] == pytest.approx(float(np.mean(fl.astype(np.float64))), rel=1e-12)
    with pytest.raises(NotImplementedError, match="auxiliary"):
        D.evaluate(feats)
