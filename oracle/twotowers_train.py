"""CPU oracle of `model.fit` for the two-tower model (neural_cf_model_2 with its final Dense, NeuralCF.py:57-70),
compiled as NeuralCF.py:74-91 compiles neural_cf_model_1: `compile(loss='binary_crossentropy', optimizer='adam')`.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

What one step computes (DESIGN.md section 4.27), in numpy at `dtype` (float32 or float64):

* forward: each tower relu(Dense) per hidden layer from its embedding row (the item tower from movieId_embedding, the
  user tower from userId_embedding), the Dot d = item . user, the final Dense z = d w_out + b_out, p = sigmoid(z)
  (`oracle.ctr_oracle.twotowers_forward`);
* loss: the logit-path binary cross-entropy, mean over the batch's rows, so dL/dz_i = (p_i - y_i) / B_batch;
* backward: dense_out's gradients dz d (kernel) and dz (bias); the Dot's gradient g = dz w_out, so the item tower's
  last delta is g hu [hi > 0] and the user tower's g hi [hu > 0]; each tower back through its hidden layers
  (relu' = [a > 0]) into its embedding row; an id that occurs several times in the batch gets the sum of its rows'
  gradients, added in row order;
* Keras Adam: `oracle.ncf_train.Adam`, both tables in the sparse (IndexedSlices) form, every Dense tensor in ApplyAdam's.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import keras_eval
from .ncf_train import KERAS_ADAM, TABLES, Adam, as_dtype, epoch_orders  # noqa: F401 (KERAS_ADAM, TABLES, epoch_orders)

SIDES = (("item", "movieId_embedding"), ("user", "userId_embedding"))


def n_layers(W) -> int:
    """Hidden layers per tower of a two-tower weight dict (item_dense_0 .. item_dense_{L-1})."""
    L = 0
    while "item_dense_%d/kernel" % L in W:
        L += 1
    return L


def forward(W, mid, uid, dtype=np.float32):
    """(p, z, cache): probabilities and logits [B]; cache = (each tower's inputs and outputs per layer, d)."""
    L = n_layers(W)
    hs = {}
    for side, table in SIDES:
        h = [np.asarray(W[table])[mid if side == "item" else uid].astype(dtype)]
        for l in range(L):
            a = h[-1] @ W["%s_dense_%d/kernel" % (side, l)].astype(dtype) \
                + W["%s_dense_%d/bias" % (side, l)].reshape(-1).astype(dtype)
            h.append(np.maximum(a, dtype(0)))
        hs[side] = h
    d = np.sum(hs["item"][-1] * hs["user"][-1], axis=1).astype(dtype)
    z = (d * W["dense_out/kernel"].reshape(-1)[0].astype(dtype) + W["dense_out/bias"].reshape(-1)[0].astype(dtype))
    z = z.astype(dtype)
    e = np.exp(-np.abs(z))                                     # stable sigmoid, both signs
    p = np.where(z >= 0, dtype(1) / (dtype(1) + e), e / (dtype(1) + e)).astype(dtype)
    return p, z, (hs, d)


def batch_loss(W, mid, uid, y, dtype=np.float64) -> float:
    """Mean over the batch of max(z,0) - z*y + log1p(exp(-|z|))."""
    _, z, _ = forward(W, mid, uid, dtype)
    yv = np.asarray(y).astype(dtype)
    return float(np.mean(np.maximum(z, 0) - z * yv + np.log1p(np.exp(-np.abs(z)))))


def gradients(W, mid, uid, y, dtype=np.float32):
    """(grads, p, z): grads in the shapes of W.  Table gradients are dense [V, E] arrays that are zero off the
    batch; a repeated id sums its rows in row order (np.add.at)."""
    p, z, (hs, d) = forward(W, mid, uid, dtype)
    B = len(mid)
    L = n_layers(W)
    dz = ((p - np.asarray(y).astype(dtype)) / dtype(B)).astype(dtype)
    g: Dict[str, np.ndarray] = {
        "dense_out/kernel": np.sum(d * dz, dtype=dtype).reshape(W["dense_out/kernel"].shape).astype(dtype),
        "dense_out/bias": np.sum(dz, dtype=dtype).reshape(W["dense_out/bias"].shape).astype(dtype)}
    gdot = (dz * W["dense_out/kernel"].reshape(-1)[0].astype(dtype)).astype(dtype)[:, None]   # [B, 1] at the Dot
    hi, hu = hs["item"][-1], hs["user"][-1]
    last = {"item": (gdot * hu) * (hi > 0), "user": (gdot * hi) * (hu > 0)}
    ids = {"item": mid, "user": uid}
    for side, table in SIDES:
        h, dl = hs[side], last[side].astype(dtype)
        for l in range(L - 1, -1, -1):
            K = W["%s_dense_%d/kernel" % (side, l)].astype(dtype)
            g["%s_dense_%d/kernel" % (side, l)] = (h[l].T @ dl).astype(dtype)
            g["%s_dense_%d/bias" % (side, l)] = dl.sum(0).astype(dtype).reshape(W["%s_dense_%d/bias" % (side, l)].shape)
            dl = (dl @ K.T).astype(dtype)
            if l > 0:
                dl = dl * (h[l] > 0)
        G = np.zeros(W[table].shape, dtype)
        np.add.at(G, np.asarray(ids[side]), dl)
        g[table] = G
    return g, p, z


def fit(W, movie, user, label, orders, batch_size: int, dtype=np.float32, hp=None, lazy: bool = False,
        max_steps: Optional[int] = None, keep_outputs: bool = False):
    """`model.fit` over the rows in `orders` [epochs][n] (each a permutation of 0..n-1), batches of `batch_size`
    consecutive entries, the last one partial.  Returns (weights at `dtype`, history, outputs, Adam), as
    `oracle.ncf_train.fit`:

    * history: per epoch `oracle.keras_eval.keras_evaluate` of that epoch's forward outputs, each taken before its
      step's update (Keras >= 2.2 `fit` logs);
    * outputs: per step (p, z, labels) when `keep_outputs`, else None.
    `max_steps` stops after that many steps in all (the last epoch's history then covers the steps it ran)."""
    W = as_dtype(W, dtype)
    opt = Adam(W, dtype, hp, lazy)
    movie, user, label = (np.asarray(a) for a in (movie, user, label))
    history: List[dict] = []
    outputs = [] if keep_outputs else None
    steps = 0
    for order in orders:
        ps, zs, ys = [], [], []
        for lo in range(0, len(order), batch_size):
            if max_steps is not None and steps >= max_steps:
                break
            rows = np.asarray(order[lo:lo + batch_size])
            mid, uid, y = movie[rows], user[rows], label[rows]
            g, p, z = gradients(W, mid, uid, y, dtype)
            opt.step(W, g, {"movieId_embedding": mid, "userId_embedding": uid})
            ps.append(p); zs.append(z); ys.append(y)
            if keep_outputs:
                outputs.append((p.copy(), z.copy(), y.copy()))
            steps += 1
        if ps:
            r = keras_eval.keras_evaluate(np.concatenate(ps).astype(np.float32),
                                          np.concatenate(zs).astype(np.float32), np.concatenate(ys))
            history.append({k: r[k] for k in ("loss", "accuracy", "roc_auc", "pr_auc")})
        if max_steps is not None and steps >= max_steps:
            break
    return W, history, outputs, opt
