"""CPU oracle of `model.fit` for DIEN, the training call of the reference's DIEN.py: `compile(optimizer="adam")`
with no compiled loss, `add_loss(final_loss)`, and `fit(train_dataset, epochs=5)` over
`from_tensor_slices(...).batch(12)` in file order (no shuffle).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

Keras 2.x behaviour restated from memory: no TensorFlow source is pinned here (DESIGN.md section 4.20).  One step,
in numpy at `dtype` (float32 or float64):

* forward: exactly `ctr_oracle.dien_forward` - the GRU consumes the Embedding mask (a step with history id 0 carries
  state and output over: where(mask, new, old)), attention s_t = sigmoid(Dense1(sigmoid(Dense32(g_t * c)))), the
  AUGRU from the stored `augru_h0`, the top MLP with PReLU - plus the auxiliary head of DESIGN.md section 4.7:
  aux_i = sum_{t>=1} pos_t + neg_t over [g_{t-1} | e(h_t)] and [g_{t-1} | e(n_t)] (0-based t), no mask;
* objective: the only loss is add_loss(final_loss), final_loss_i = bce_i - 0.5 * mean_j(aux_j); tape.gradient of
  the non-scalar target differentiates its SUM over the batch, so dL/dz_i = sigmoid(z_i) - y_i (no 1/B) and every
  pos_t / neg_t gets -0.5.  That raises both auxiliary probabilities: the script as written;
* backward: BPTT through GRU (reset_after, z | r | h; a masked step passes dh through and adds nothing), attention,
  AUGRU and the auxiliary head; PReLU's delta up * ([x > 0] + alpha [x < 0]) and dalpha = up * min(x, 0);
  `embedding` collects the candidate, every history position (the GRU's input gradient and the head's) and every
  negative; an id repeated in a batch sums its entries (np.add.at);
* `augru_h0` is not a variable in the reference (a fresh draw inside `call`): its gradient is zero, so Adam leaves
  it bit for bit;
* Keras Adam (`deepfm_train.Adam`'s formulas): the four tables take the sparse form on every row, every other tensor
  ApplyAdam's dense form.

`defect` (mutants for the tests): "mask" ignores the mask in BPTT, "h0" trains augru_h0, "aux" drops the auxiliary
head's gradient, "step" drops position 0's gradients, "mean" divides the objective by B, "last" gives the embedding
rows of history position T - 1 no gradient.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import deepfm_train, keras_eval
from .ctr_oracle import sigmoid

TABLES = ("embedding", "userId_embedding", "userGenre1_embedding", "movieGenre1_embedding")
NUMERIC_KEYS = ("movieAvgRating", "movieRatingCount", "movieRatingStddev", "releaseYear", "userAvgRating",
                "userRatingCount", "userRatingStddev")
GATES = ("r", "z", "h")


class Adam(deepfm_train.Adam):
    """Keras Adam over DIEN's variables, the four tables of TABLES in the sparse form."""

    TABLES = TABLES


class Rows:
    """The columns one DIEN step reads: candidate, user, genre indices (-1 = missing), the 7 numerics (NUMERIC_KEYS
    order), history ids [B, T] in graph order, negatives [B, T - 1], labels."""

    def __init__(self, mid, uid, ig, ug, num, hist, neg, y=None):
        self.mid, self.uid, self.ig, self.ug = (np.asarray(a, np.int64) for a in (mid, uid, ig, ug))
        self.num = np.asarray(num, np.float32)
        self.hist = np.asarray(hist, np.int64)
        self.neg = np.asarray(neg, np.int64).reshape(len(self.mid), -1)
        self.y = None if y is None else np.asarray(y)

    @classmethod
    def from_features(cls, feats, T) -> "Rows":
        """From a feature dict (genres as vocabulary indices, `negtive_userRatedMovie2..T`, "label")."""
        from .ctr_oracle import din_history_keys, genre_index
        num = np.stack([np.asarray(feats[k]).astype(np.float32) for k in NUMERIC_KEYS], axis=1)
        hist = np.stack([np.asarray(feats[k]).astype(np.float32).astype(np.int64) for k in din_history_keys(T)], 1)
        neg = np.stack([np.asarray(feats["negtive_userRatedMovie%d" % k]).astype(np.float32).astype(np.int64)
                        for k in range(2, T + 1)], 1) if T > 1 else np.zeros((len(num), 0), np.int64)
        return cls(np.asarray(feats["movieId"]).astype(np.float32).astype(np.int64), feats["userId"],
                   genre_index(feats, "movieGenre1"), genre_index(feats, "userGenre1"), num, hist, neg,
                   feats.get("label"))

    def take(self, rows) -> "Rows":
        return Rows(self.mid[rows], self.uid[rows], self.ig[rows], self.ug[rows], self.num[rows], self.hist[rows],
                    self.neg[rows], None if self.y is None else self.y[rows])


def _lookup(table, ids, dtype):
    out = table.astype(dtype)[np.maximum(ids, 0)]
    out[ids < 0] = 0
    return out


def forward(W, r: Rows, dtype=np.float32):
    """(p, z, aux, cache): probabilities, logits and aux [B], and what backward needs."""
    dt = dtype
    w = {k: v.astype(dt) for k, v in W.items()}
    B, T = r.hist.shape
    E = w["embedding"].shape[1]
    tab = w["embedding"]
    X, C = tab[r.hist], tab[r.mid]
    mask = r.hist != 0
    K, U = w["gru/kernel"], w["gru_recurrent/kernel"]
    bx, bh = w["gru/bias"]
    h = np.zeros((B, E), dt)
    G, gru = np.zeros((B, T, E), dt), []
    for t in range(T):
        mx = X[:, t] @ K + bx
        mh = h @ U + bh
        z = sigmoid(mx[:, :E] + mh[:, :E])
        rg = sigmoid(mx[:, E:2 * E] + mh[:, E:2 * E])
        hh = np.tanh(mx[:, 2 * E:] + rg * mh[:, 2 * E:])
        gru.append(dict(hp=h, z=z, r=rg, hh=hh, rh=mh[:, 2 * E:]))
        h = np.where(mask[:, t, None], z * h + (1 - z) * hh, h).astype(dt)
        G[:, t] = h
    heads = []
    aux = np.zeros(B, dt)
    for t in range(1, T):
        d = {}
        for side, e in (("pos", X[:, t]), ("neg", tab[r.neg[:, t - 1]])):
            x = np.concatenate([G[:, t - 1], e], axis=1)
            sp = sigmoid(x @ w["aux_%s_dense/kernel" % side] + w["aux_%s_dense/bias" % side])
            o = sigmoid(sp @ w["aux_%s_out/kernel" % side] + w["aux_%s_out/bias" % side])[:, 0]
            d[side] = dict(x=x, sp=sp, o=o)
            aux = aux + o
        heads.append(d)
    PC = G * C[:, None, :]
    A = sigmoid(PC @ w["att_dense/kernel"] + w["att_dense/bias"])
    S = sigmoid(A @ w["att_out/kernel"] + w["att_out/bias"])[..., 0]
    u = np.repeat(w["augru_h0"], B, axis=0)
    aug = []
    for t in range(T):
        x = G[:, t]
        c = dict(up=u)
        for g in ("r", "z"):
            c["p" + g] = x @ w["augru_%s_input/kernel" % g] + w["augru_%s_input/bias" % g] + \
                u @ w["augru_%s_hidden/kernel" % g]
            c[g] = sigmoid(c["p" + g] @ w["augru_%s_act/kernel" % g] + w["augru_%s_act/bias" % g])
        c["uz"] = u * c["z"]
        c["ph"] = x @ w["augru_h_input/kernel"] + w["augru_h_input/bias"] + c["uz"] @ w["augru_h_hidden/kernel"]
        c["hn"] = np.tanh(c["ph"] @ w["augru_h_act/kernel"] + w["augru_h_act/bias"])
        c["ra"] = S[:, t, None] * c["r"]
        u = ((1 - c["ra"]) * u + c["ra"] * c["hn"]).astype(dt)
        aug.append(c)
    num = r.num.astype(dt)
    up = np.concatenate([num[:, 4:5], _lookup(w["userGenre1_embedding"], r.ug, dt),
                         _lookup(w["userId_embedding"], r.uid, dt), num[:, 5:7]], axis=1)
    ctx = np.concatenate([num[:, 0:1], _lookup(w["movieGenre1_embedding"], r.ig, dt), num[:, 1:4]], axis=1)
    x0 = np.concatenate([u, C, up, ctx], axis=1)
    P1 = x0 @ w["dense/kernel"] + w["dense/bias"]
    H1 = np.where(P1 > 0, P1, w["prelu/alpha"] * P1)
    P2 = H1 @ w["dense_1/kernel"] + w["dense_1/bias"]
    H2 = np.where(P2 > 0, P2, w["prelu_1/alpha"] * P2)
    z = (H2 @ w["dense_2/kernel"] + w["dense_2/bias"])[:, 0]
    e = np.exp(-np.abs(z))
    p = np.where(z >= 0, 1 / (1 + e), e / (1 + e)).astype(dt)
    return p, z, aux, dict(w=w, X=X, C=C, mask=mask, G=G, gru=gru, heads=heads, PC=PC, A=A, S=S, aug=aug, x0=x0,
                           P1=P1, H1=H1, P2=P2, H2=H2, E=E)


def _prelu_delta(up, x, alpha):
    return up * ((x > 0) + alpha * (x < 0))


def gradients(W, r: Rows, y, dtype=np.float32, defect: Optional[str] = None):
    """(grads, p, z, aux): grads in the shapes of W (tables dense, zero off the batch)."""
    p, z, aux, c = forward(W, r, dtype)
    w, E, dt = c["w"], c["E"], dtype
    B, T = r.hist.shape
    g: Dict[str, np.ndarray] = {k: np.zeros(v.shape, dt) for k, v in W.items()}
    dz = (p - np.asarray(y).astype(dt)).astype(dt)
    daux = dt(-0.5)
    if defect == "mean":
        dz, daux = dz / dt(B), daux / dt(B)
    if defect == "aux":
        daux = dt(0)
    # top MLP
    g["dense_2/kernel"] = (c["H2"].T @ dz)[:, None]
    g["dense_2/bias"] = np.array([dz.sum()], dt)
    up2 = dz[:, None] * w["dense_2/kernel"][:, 0]
    g["prelu_1/alpha"] = (up2 * np.minimum(c["P2"], 0)).sum(0)
    d2 = _prelu_delta(up2, c["P2"], w["prelu_1/alpha"])
    g["dense_1/kernel"] = c["H1"].T @ d2
    g["dense_1/bias"] = d2.sum(0)
    up1 = d2 @ w["dense_1/kernel"].T
    g["prelu/alpha"] = (up1 * np.minimum(c["P1"], 0)).sum(0)
    d1 = _prelu_delta(up1, c["P1"], w["prelu/alpha"])
    g["dense/kernel"] = c["x0"].T @ d1
    g["dense/bias"] = d1.sum(0)
    dx0 = d1 @ w["dense/kernel"].T
    du = dx0[:, :E]
    dC = dx0[:, E:2 * E].copy()
    gt = dx0[:, 2 * E:]                      # [userAvgRating | ug E | uid E | 2 | movieAvgRating | ig E | 3]
    G_ug, G_uid, G_ig = gt[:, 1:1 + E], gt[:, 1 + E:1 + 2 * E], gt[:, 3 + 2 * E + 1:3 + 3 * E + 1]
    ok = r.ug >= 0
    np.add.at(g["userGenre1_embedding"], r.ug[ok], G_ug[ok])
    np.add.at(g["userId_embedding"], r.uid, G_uid)
    ok = r.ig >= 0
    np.add.at(g["movieGenre1_embedding"], r.ig[ok], G_ig[ok])
    # AUGRU and attention, t = T-1 .. 0
    dG = np.zeros((B, T, E), dt)
    dS = np.zeros((B, T), dt)
    for t in range(T - 1, -1, -1):
        a = c["aug"][t]
        x = c["G"][:, t]
        d_ra = du * (a["hn"] - a["up"])
        d_hn = du * a["ra"]
        du_p = du * (1 - a["ra"])
        dS[:, t] = (d_ra * a["r"]).sum(1)
        d_rg = d_ra * c["S"][:, t, None]
        d_ah = d_hn * (1 - a["hn"] ** 2)
        g["augru_h_act/kernel"] += a["ph"].T @ d_ah
        g["augru_h_act/bias"] += d_ah.sum(0)
        d_ph = d_ah @ w["augru_h_act/kernel"].T
        g["augru_h_input/kernel"] += x.T @ d_ph
        g["augru_h_input/bias"] += d_ph.sum(0)
        g["augru_h_hidden/kernel"] += a["uz"].T @ d_ph
        d_uz = d_ph @ w["augru_h_hidden/kernel"].T
        du_p = du_p + d_uz * a["z"]
        d_zg = d_uz * a["up"]
        dx = d_ph @ w["augru_h_input/kernel"].T
        for gg, dgate in (("r", d_rg), ("z", d_zg)):
            d_act = dgate * a[gg] * (1 - a[gg])
            g["augru_%s_act/kernel" % gg] += a["p" + gg].T @ d_act
            g["augru_%s_act/bias" % gg] += d_act.sum(0)
            d_p = d_act @ w["augru_%s_act/kernel" % gg].T
            g["augru_%s_input/kernel" % gg] += x.T @ d_p
            g["augru_%s_input/bias" % gg] += d_p.sum(0)
            g["augru_%s_hidden/kernel" % gg] += a["up"].T @ d_p
            du_p = du_p + d_p @ w["augru_%s_hidden/kernel" % gg].T
            dx = dx + d_p @ w["augru_%s_input/kernel" % gg].T
        dG[:, t] += dx
        du = du_p
    if defect == "h0":
        g["augru_h0"] = du.sum(0)[None, :]
    d_sz = dS * c["S"] * (1 - c["S"])                           # [B, T]
    g["att_out/kernel"] = np.einsum("btj,bt->j", c["A"], d_sz)[:, None]
    g["att_out/bias"] = np.array([d_sz.sum()], dt)
    d_at = d_sz[..., None] * w["att_out/kernel"][:, 0] * c["A"] * (1 - c["A"])
    g["att_dense/kernel"] = np.einsum("btk,btj->kj", c["PC"], d_at)
    g["att_dense/bias"] = d_at.sum((0, 1))
    d_pc = d_at @ w["att_dense/kernel"].T
    dG += d_pc * c["C"][:, None, :]
    dC += (d_pc * c["G"]).sum(1)
    # the auxiliary head: g_{t-1}, e(h_t), e(n_t)
    dX = np.zeros((B, T, E), dt)
    dN = np.zeros((B, max(T - 1, 0), E), dt)
    for t in range(1, T):
        for side in ("pos", "neg"):
            hd = c["heads"][t - 1][side]
            d_o = daux * hd["o"] * (1 - hd["o"])
            g["aux_%s_out/kernel" % side] += (hd["sp"].T @ d_o)[:, None]
            g["aux_%s_out/bias" % side] += d_o.sum()
            d_a = d_o[:, None] * w["aux_%s_out/kernel" % side][:, 0] * hd["sp"] * (1 - hd["sp"])
            g["aux_%s_dense/kernel" % side] += hd["x"].T @ d_a
            g["aux_%s_dense/bias" % side] += d_a.sum(0)
            dxa = d_a @ w["aux_%s_dense/kernel" % side].T
            dG[:, t - 1] += dxa[:, :E]
            if side == "pos":
                dX[:, t] += dxa[:, E:]
            else:
                dN[:, t - 1] += dxa[:, E:]
    # GRU BPTT
    K, U = w["gru/kernel"], w["gru_recurrent/kernel"]
    dh = np.zeros((B, E), dt)
    t_end = 1 if defect == "step" else 0
    for t in range(T - 1, t_end - 1, -1):
        q = c["gru"][t]
        dh = dh + dG[:, t]
        m = c["mask"][:, t, None] if defect != "mask" else np.ones((B, 1), bool)
        d_z = dh * (q["hp"] - q["hh"])
        d_hh = dh * (1 - q["z"])
        dxh = d_hh * (1 - q["hh"] ** 2)
        drh = dxh * q["r"]
        dxr = dxh * q["rh"] * q["r"] * (1 - q["r"])
        dxz = d_z * q["z"] * (1 - q["z"])
        dmx = np.where(m, np.concatenate([dxz, dxr, dxh], 1), 0).astype(dt)
        dmh = np.where(m, np.concatenate([dxz, dxr, drh], 1), 0).astype(dt)
        g["gru/kernel"] += c["X"][:, t].T @ dmx
        g["gru_recurrent/kernel"] += q["hp"].T @ dmh
        g["gru/bias"][0] += dmx.sum(0)
        g["gru/bias"][1] += dmh.sum(0)
        dX[:, t] += dmx @ K.T
        dh = np.where(m, dh * q["z"] + dmh @ U.T, dh).astype(dt)
    emb = g["embedding"]
    np.add.at(emb, r.mid, dC)
    for t in range(T - 1 if defect == "last" else T):
        np.add.at(emb, r.hist[:, t], dX[:, t])
    for t in range(1, T):
        np.add.at(emb, r.neg[:, t - 1], dN[:, t - 1])
    g = {k: v.reshape(W[k].shape).astype(dt) for k, v in g.items()}
    return g, p, z, aux


def final_loss(z, y, aux) -> np.ndarray:
    """DIEN.py:287 for one batch: bce_i (float32 logit path) - 0.5 * mean(aux), in float64."""
    bce = keras_eval.logit_bce_f32(np.asarray(z, np.float32), np.asarray(y)).astype(np.float64)
    return bce - 0.5 * np.mean(np.asarray(aux, np.float64))


def history_entry(ps, zs, ys, auxs) -> dict:
    """{"loss", "auc", "auc_value"} of an epoch's steps, as srs_dien_eval_result defines them."""
    n = sum(len(p) for p in ps)
    loss = sum(final_loss(z, y, a).sum() for z, y, a in zip(zs, ys, auxs)) / n
    aucs, acc = [], None                       # the counts of batches 0..k, added batch by batch
    for p, y in zip(ps, ys):
        c = keras_eval.confusion_counts(np.asarray(p, np.float32), y)
        acc = c if acc is None else tuple(a + b for a, b in zip(acc, c))
        aucs.append(keras_eval.roc_auc_from_counts(*acc))
    return {"loss": float(loss), "auc": aucs[-1], "auc_value": float(np.mean(aucs))}


def fit(W, data: Rows, orders, batch_size: int, dtype=np.float32, hp=None, lazy: bool = False,
        max_steps: Optional[int] = None, defect: Optional[str] = None):
    """`model.fit` over the rows in `orders` [epochs][n] (the script's: file order), batches of `batch_size`
    consecutive entries, the last one partial.  Returns (weights at `dtype`, history, Adam)."""
    W = {k: np.array(v, dtype) for k, v in W.items()}
    opt = Adam(W, dtype, hp, lazy)
    history: List[dict] = []
    steps = 0
    for order in orders:
        ps, zs, ys, auxs = [], [], [], []
        for lo in range(0, len(order), batch_size):
            if max_steps is not None and steps >= max_steps:
                break
            rows = np.asarray(order[lo:lo + batch_size])
            r = data.take(rows)
            g, p, z, aux = gradients(W, r, r.y, dtype, defect)
            rows_of = {"embedding": np.concatenate([r.mid, r.hist.ravel(), r.neg.ravel()]),
                       "userId_embedding": r.uid, "userGenre1_embedding": r.ug[r.ug >= 0],
                       "movieGenre1_embedding": r.ig[r.ig >= 0]}
            opt.step(W, g, rows_of)
            ps.append(p); zs.append(z); ys.append(np.asarray(r.y)); auxs.append(aux)
            steps += 1
        if ps:
            history.append(history_entry(ps, zs, ys, auxs))
        if max_steps is not None and steps >= max_steps:
            break
    return W, history, opt
