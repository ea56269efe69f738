"""CPU oracle of `model.fit` for NeuralCF (neural_cf_model_1), the training call of the reference's
NeuralCF.py:74-91: `compile(loss='binary_crossentropy', optimizer='adam')` and `fit(train_dataset, epochs=5)`.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

What one step computes (DESIGN.md section 4.8), in numpy at `dtype` (float32 or float64):

* forward: x = [movieEmb | userEmb], relu(Dense) per hidden layer, Dense 1 -> logit z, p = sigmoid(z);
* loss: the logit-path binary cross-entropy, mean over the batch's rows, so dL/dz_i = (p_i - y_i) / B_batch;
* backward through the Dense layers (relu' = [a > 0]) into the two embedding rows of each row; an id that occurs
  several times in the batch gets the sum of its rows' gradients, added in row order;
* Keras Adam (restated from memory of TF 2.x's optimizer_v2/adam.py and the fused ApplyAdam kernel, as the rest of
  DESIGN section 2): t = iterations + 1, alpha = lr * sqrt(1 - beta_2^t) / (1 - beta_1^t);
    Dense kernels / biases (ApplyAdam):  m += (g - m)(1 - beta_1);  v += (g*g - v)(1 - beta_2)
    embedding tables (_resource_apply_sparse, IndexedSlices): m = beta_1 m + (1 - beta_1) G;
                                         v = beta_2 v + (1 - beta_2) G*G     on EVERY row (G = 0 off the batch)
    both:                                w -= alpha m / (sqrt(v) + epsilon)  on every element.
  `lazy=True` restates "lazy Adam" instead (only the batch's table rows move); it exists so that a test can tell
  the two apart.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import keras_eval

TABLES = ("movieId_embedding", "userId_embedding")
KERAS_ADAM = {"lr": 0.001, "beta_1": 0.9, "beta_2": 0.999, "epsilon": 1e-7}


def n_layers(W) -> int:
    """Hidden layers of a NeuralCF weight dict (dense_0 .. dense_{L-1} hidden, dense_L the output)."""
    L = 0
    while "dense_%d/kernel" % (L + 1) in W:
        L += 1
    return L


def forward(W, mid, uid, dtype=np.float32):
    """(p, z, cache): probabilities and logits [B] and what backward needs."""
    x = np.concatenate([W["movieId_embedding"][mid], W["userId_embedding"][uid]], axis=1).astype(dtype)
    L = n_layers(W)
    hs = [x]
    for l in range(L):
        a = hs[-1] @ W["dense_%d/kernel" % l].astype(dtype) + W["dense_%d/bias" % l].reshape(-1).astype(dtype)
        hs.append(np.maximum(a, dtype(0)))
    z = (hs[-1] @ W["dense_%d/kernel" % L].astype(dtype))[:, 0] + W["dense_%d/bias" % L].reshape(-1)[0].astype(dtype)
    z = z.astype(dtype)
    e = np.exp(-np.abs(z))                                     # stable sigmoid, both signs
    p = np.where(z >= 0, dtype(1) / (dtype(1) + e), e / (dtype(1) + e)).astype(dtype)
    return p, z, hs


def batch_loss(W, mid, uid, y, dtype=np.float64) -> float:
    """Mean over the batch of max(z,0) - z*y + log1p(exp(-|z|))."""
    _, z, _ = forward(W, mid, uid, dtype)
    yv = np.asarray(y).astype(dtype)
    return float(np.mean(np.maximum(z, 0) - z * yv + np.log1p(np.exp(-np.abs(z)))))


def gradients(W, mid, uid, y, dtype=np.float32):
    """(grads, p, z): grads in the shapes of W.  Table gradients are dense [V, E] arrays that are zero off the
    batch; a repeated id sums its rows in row order (np.add.at)."""
    p, z, hs = forward(W, mid, uid, dtype)
    B = len(mid)
    L = n_layers(W)
    dz = ((p - np.asarray(y).astype(dtype)) / dtype(B)).astype(dtype)
    g: Dict[str, np.ndarray] = {}
    d = dz[:, None]                                           # [B, 1] gradient at the output pre-activation
    for l in range(L, -1, -1):
        K = W["dense_%d/kernel" % l].astype(dtype)
        g["dense_%d/kernel" % l] = (hs[l].T @ d).astype(dtype)
        g["dense_%d/bias" % l] = d.sum(0).astype(dtype).reshape(W["dense_%d/bias" % l].shape)
        d = (d @ K.T).astype(dtype)
        if l > 0:
            d = d * (hs[l] > 0)
    E = W["movieId_embedding"].shape[1]
    for name, ids, part in (("movieId_embedding", mid, d[:, :E]), ("userId_embedding", uid, d[:, E:])):
        G = np.zeros(W[name].shape, dtype)
        np.add.at(G, np.asarray(ids), part)
        g[name] = G
    return g, p, z


class Adam:
    """Keras Adam state: m, v per tensor and the iteration count."""

    def __init__(self, W, dtype=np.float32, hp: Optional[dict] = None, lazy: bool = False):
        self.dtype = dtype
        self.hp = dict(KERAS_ADAM, **(hp or {}))
        self.m = {k: np.zeros(v.shape, dtype) for k, v in W.items()}
        self.v = {k: np.zeros(v.shape, dtype) for k, v in W.items()}
        self.iterations = 0
        self.lazy = lazy

    def step(self, W, g, rows=None):
        """Update W in place with gradients g.  `rows` (lazy Adam only): {table name: ids of the batch}."""
        dt = self.dtype
        b1, b2 = dt(self.hp["beta_1"]), dt(self.hp["beta_2"])
        eps, lr = dt(self.hp["epsilon"]), dt(self.hp["lr"])
        t = dt(self.iterations + 1)
        alpha = dt(lr * (np.sqrt(dt(1) - b2 ** t) / (dt(1) - b1 ** t)))
        one_b1, one_b2 = dt(1) - b1, dt(1) - b2
        for k in W:
            m, v, gk = self.m[k], self.v[k], g[k].astype(dt)
            if k in TABLES:
                if self.lazy:
                    r = np.unique(rows[k])
                    m[r] = b1 * m[r] + one_b1 * gk[r]
                    v[r] = b2 * v[r] + one_b2 * (gk[r] * gk[r])
                    W[k][r] = (W[k][r] - (alpha * m[r]) / (np.sqrt(v[r]) + eps)).astype(W[k].dtype)
                    continue
                m[...] = b1 * m + one_b1 * gk
                v[...] = b2 * v + one_b2 * (gk * gk)
            else:
                m += (gk - m) * one_b1
                v += (gk * gk - v) * one_b2
            W[k][...] = W[k] - (alpha * m) / (np.sqrt(v) + eps)
        self.iterations += 1


def as_dtype(W, dtype):
    return {k: np.array(v, dtype) for k, v in W.items()}


def fit(W, movie, user, label, orders, batch_size: int, dtype=np.float32, hp=None, lazy: bool = False,
        max_steps: Optional[int] = None, keep_outputs: bool = False):
    """`model.fit` over the rows in `orders` [epochs][n] (each a permutation of 0..n-1), batches of `batch_size`
    consecutive entries, the last one partial.  Returns (weights at `dtype`, history, outputs):

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


def epoch_orders(n: int, epochs: int, seed: int) -> np.ndarray:
    """The row order `Trainer.fit` uses: one `numpy.random.default_rng(seed).permutation(n)` per epoch."""
    rng = np.random.default_rng(seed)
    return np.stack([rng.permutation(n) for _ in range(epochs)]).astype(np.int32)
