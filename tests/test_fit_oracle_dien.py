"""CPU checks of DIEN's training oracle (oracle/dien_train.py, DESIGN.md section 4.20) and of the trainer's
device-free rejections."""
import ctypes as C

import numpy as np
import pytest

from oracle import ctr_oracle, dien_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_aux_weights, init_weights


def _case(E, T, n, seed, n_movies=30):
    from sparrowrecsys_b200.features import negative_history, synthetic_features
    spec = default_spec("dien", emb_dim=E, hist_len=T, n_movies=n_movies, n_users=20, hidden=(6, 5))
    W = {**init_weights(spec, seed), **init_aux_weights(spec, seed)}
    rng = np.random.default_rng(seed)
    for k in W:
        if k.endswith("/bias") or k.endswith("/alpha"):
            W[k] = rng.uniform(-0.3, 0.3, W[k].shape).astype(np.float32)
    f = synthetic_features(spec, n, seed=seed)
    for k in dien_train.NUMERIC_KEYS:       # unit-scale numerics: a finite difference stays off the PReLU kinks
        f[k] = rng.uniform(0, 1, n).astype(np.float32)
    keys = ctr_oracle.din_history_keys(T)
    for k in keys:
        f[k] = np.array(f[k])
    if T > 1 and n > 3:                     # padding at the start, the middle and the end of a history
        f[keys[0]][0] = 0
        f[keys[T // 2]][1] = 0
        f[keys[-1]][2] = 0
    if n > 4:
        for k in keys:                      # an all-padding history
            f[k][3] = 0
        f["movieId"] = np.array(f["movieId"])
        f["movieId"][4] = f[keys[0]][4]     # a candidate among its own history
    for g in ("movieGenre1", "userGenre1"):
        f[g] = np.array(f[g], dtype=object)
        f[g][::3] = ""                      # missing genres
    f.update(negative_history(f, T, seed, n_movies=n_movies))
    if T > 1 and n > 5:                     # a negative that is another row's positive
        f["negtive_userRatedMovie2"] = np.array(f["negtive_userRatedMovie2"])
        f["negtive_userRatedMovie2"][5] = f[keys[1]][0]
    f["label"] = (rng.random(n) < 0.5).astype(np.int32)
    return spec, W, f


def _objective(W, r):
    _, z, aux, _ = dien_train.forward(W, r, np.float64)
    y = r.y.astype(np.float64)
    return float((np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z))) - 0.5 * aux.mean()).sum())


def test_forward_is_dien_forward_and_aux_is_the_head():
    spec, W, f = _case(5, 4, 9, 1)
    r = dien_train.Rows.from_features(f, 4)
    p, z, aux, c = dien_train.forward(W, r, np.float64)
    p0, z0 = ctr_oracle.dien_forward(spec, W, f, np.float64)
    assert np.abs(z - z0[:, 0]).max() <= 1e-12 and np.abs(p - p0[:, 0]).max() <= 1e-12
    # the head as a per-row, per-position loop (DIEN.py:276-285)
    sig = lambda v: 1 / (1 + np.exp(-v))
    w = {k: v.astype(np.float64) for k, v in W.items()}
    tab = w["embedding"]
    for i in range(len(z)):
        want = 0.0
        for t in range(1, 4):
            for side, e in (("pos", tab[r.hist[i, t]]), ("neg", tab[r.neg[i, t - 1]])):
                x = np.concatenate([c["G"][i, t - 1], e])
                hid = sig(x @ w["aux_%s_dense/kernel" % side] + w["aux_%s_dense/bias" % side])
                want += sig(hid @ w["aux_%s_out/kernel" % side][:, 0] + w["aux_%s_out/bias" % side][0])
        assert abs(aux[i] - want) <= 1e-12


@pytest.mark.parametrize("E,T,n", [(5, 4, 7), (3, 1, 5), (4, 2, 6), (2, 3, 1)])
def test_gradients_match_central_differences_for_every_tensor(E, T, n):
    spec, W, f = _case(E, T, n, E + T)
    r = dien_train.Rows.from_features(f, T)
    g, _, _, _ = dien_train.gradients(W, r, r.y, np.float64)
    W64 = {k: v.astype(np.float64) for k, v in W.items()}
    rng = np.random.default_rng(0)
    for k in W64:
        idx = list(np.ndindex(W64[k].shape))
        if len(idx) > 24:
            idx = [idx[i] for i in rng.choice(len(idx), 24, replace=False)]
        if k == "embedding":                # every id the batch touches, padding row 0 included
            idx = sorted({(int(i), j) for i in np.concatenate([r.mid, r.hist.ravel(), r.neg.ravel()])
                          for j in range(E)})
        for i in idx:
            Wp, Wm = dict(W64), dict(W64)
            Wp[k], Wm[k] = W64[k].copy(), W64[k].copy()
            Wp[k][i] += 1e-6
            Wm[k][i] -= 1e-6
            num = (_objective(Wp, r) - _objective(Wm, r)) / 2e-6
            if k == "augru_h0":             # not a variable: no gradient although the loss depends on it
                assert g[k][i] == 0.0
                continue
            assert abs(num - g[k][i]) <= 1e-6 * max(1.0, abs(num)), (k, i, num, g[k][i])
    if (r.hist[:, 1:] == 0).any():          # a padded position t >= 1: row 0 trains through the head
        assert np.abs(g["embedding"][0]).max() > 0


def test_adam_known_answers_in_both_forms():
    """Two steps from w = 1 with g = 0.7, then g = -0.61.  Step 1 starts from zero moments, where the two forms
    agree; step 2 starts from m = 0.07, v = 0.00049, where they round differently, so each form's known answer is
    checked at float32 on a table (the sparse form) and a Dense tensor (ApplyAdam's form)."""
    spec, W, f = _case(2, 2, 1, 0)
    W = {k: np.ones_like(v) for k, v in W.items()}
    f32 = np.float32
    opt = dien_train.Adam(W, f32)
    Wn = {k: v.astype(f32) for k, v in W.items()}
    for gv in (0.7, -0.61):
        opt.step(Wn, {k: np.full(v.shape, gv, f32) for k, v in W.items()})
    b1, b2, lr, eps = f32(0.9), f32(0.999), f32(0.001), f32(1e-7)
    one_b1, one_b2 = f32(1) - b1, f32(1) - b2

    def known(sparse):
        w, m, v = f32(1), f32(0), f32(0)
        for t, g in ((1, f32(0.7)), (2, f32(-0.61))):
            alpha = f32(lr * (np.sqrt(f32(1) - b2 ** f32(t)) / (f32(1) - b1 ** f32(t))))
            if sparse:
                m, v = f32(b1 * m + one_b1 * g), f32(b2 * v + one_b2 * (g * g))
            else:
                m, v = f32(m + (g - m) * one_b1), f32(v + (g * g - v) * one_b2)
            w = f32(w - (alpha * m) / (np.sqrt(v) + eps))
        return w, m, v

    ws, ms, vs = known(True)
    wd, md, vd = known(False)
    assert (ms, vs) != (md, vd)              # the second step tells the two forms apart
    assert opt.m["embedding"][0, 0] == ms and opt.v["embedding"][0, 0] == vs and Wn["embedding"][0, 0] == ws
    assert opt.m["gru/kernel"][0, 0] == md and opt.v["gru/kernel"][0, 0] == vd and Wn["gru/kernel"][0, 0] == wd
    assert opt.iterations == 2


DEFECTS = ("mask", "h0", "aux", "step", "lazy", "mean")


def test_the_parity_tolerance_catches_each_defect():
    """On the float64 oracle after 3 steps of 6 rows: every tensor but augru_h0 trains past the GPU tolerance (4x the
    float32 spread + one ulp), and each defect moves some tensor past it.  The mean in place of the sum is caught
    too, although Adam is nearly invariant to the gradient's scale: m / (sqrt(v) + epsilon) drops the scale only up
    to epsilon's share, and after 3 steps the float32 spread, hence the tolerance, is smaller than that share."""
    spec, W, f = _case(5, 4, 18, 7)
    r = dien_train.Rows.from_features(f, 4)
    orders = [np.arange(18)]
    w64, _, _ = dien_train.fit(W, r, orders, 6, np.float64)
    w32, _, _ = dien_train.fit(W, r, orders, 6, np.float32)
    tol = {k: 4 * np.abs(w32[k] - w64[k]).max() + np.spacing(np.float32(np.abs(w64[k]).max())) for k in W}
    # every tensor but augru_h0 trains past its tolerance, so no tolerance is vacuous
    still = [k for k in W if np.abs(w64[k] - W[k]).max() <= tol[k]]
    assert still == ["augru_h0"], still
    caught = {}
    for d in DEFECTS:
        wd, _, _ = dien_train.fit(W, r, orders, 6, np.float64, lazy=d == "lazy", defect=None if d == "lazy" else d)
        caught[d] = [k for k in W if np.abs(wd[k] - w64[k]).max() > tol[k]]
    for d in DEFECTS:
        assert caught[d], d
    assert "augru_h0" in caught["h0"] and "gru/kernel" in caught["mask"] and "aux_pos_dense/kernel" in caught["aux"]
    assert "embedding" in caught["mean"] and "dense/kernel" in caught["mean"]


def _lib_or_skip():
    from sparrowrecsys_b200 import _lib
    try:
        return _lib, _lib.load()
    except ImportError as e:
        pytest.skip(str(e))


@pytest.mark.parametrize("fields,match", [(dict(emb_dim=33), b"1..32"), (dict(hist_len=65), b"hist_len"),
                                          (dict(hist_len=0), b"hist_len"), (dict(au_hidden=16), b"au_hidden"),
                                          (dict(hidden=(129, 64)), b"1..128"), (dict(n_hidden=1), b"exactly 2")])
def test_create_any_rejects_unsupported_dien_shapes(fields, match):
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    sp = _spec_struct(default_spec("dien"))
    for k, v in fields.items():
        if k == "hidden":
            sp.hidden[0], sp.hidden[1] = v
        else:
            setattr(sp, k, v)
    out = C.c_void_p()
    assert lib.srs_trainer_create_any(C.byref(sp), None, 0, 0, None, C.byref(out)) == _lib.SRS_ERR_INVALID
    assert not out.value and match in lib.srs_last_error()


def test_create_and_create_ex_keep_their_lists_and_fit_dien_needs_a_trainer():
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    from sparrowrecsys_b200.training import Trainer
    assert "dien" in Trainer.MODELS
    sp = _spec_struct(default_spec("dien"))
    out = C.c_void_p()
    assert lib.srs_trainer_create(C.byref(sp), None, 0, 0, None, C.byref(out)) == _lib.SRS_ERR_INVALID
    assert lib.srs_trainer_create_ex(C.byref(sp), None, 0, 0, None, C.byref(out)) == _lib.SRS_ERR_INVALID
    assert lib.srs_trainer_fit_dien_host(None, None, None, 0, None, None, 12, 1, None) == _lib.SRS_ERR_INVALID


def test_trainer_refuses_dien_validation_without_a_device():
    from sparrowrecsys_b200.training import Trainer
    t = Trainer.__new__(Trainer)
    t.spec = default_spec("dien")
    with pytest.raises(NotImplementedError):
        t.fit({}, validation_data=({}, None))
    with pytest.raises(NotImplementedError, match="dien_evaluate"):
        t.evaluate({})
