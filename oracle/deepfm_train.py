"""CPU oracle of `model.fit` for DeepFM, the training call of the reference's DeepFM.py:
`compile(loss='binary_crossentropy', optimizer='adam', ...)` and `fit(train_dataset, epochs=5)`.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

What one step computes (DESIGN.md section 4.9), in numpy at `dtype` (float32 or float64), statement by statement
like oracle/ncf_train.py:

* forward: `ctr_oracle.deepfm_forward` - the four FM rows (item, user, movie genre, user genre; a missing genre,
  index -1, is a zero row), the dots <item,user> <ig,ug> <ig,user> <item,ug>, the deep input (the sorted
  DenseFeatures concat of the 7 numerics and the two deep rows) through Dense(relu) -> Dense(relu), and dense_2
  over [one-hots (movieGenre1 | movieId | userGenre1 | userId) | 4 dots | deep] -> logit z, p = sigmoid(z);
* loss: the logit-path binary cross-entropy, mean over the batch, so dL/dz_i = (p_i - y_i) / B_batch;
* backward: dense_2's one-hot rows get dz at the 4 rows each example selects (none for a missing genre), its dot
  rows dz . dot_d, its deep rows dz . h2; each FM row dz * sum(dot weight * the other factor); the deep MLP with
  relu' = [a > 0] into dense, dense_1 and the two deep rows.  An id that repeats within a batch gets the sum of
  its rows' gradients, in row order;
* Keras Adam (`Adam`, `ncf_train.Adam`'s state and formulas with DeepFM's variables): the six tables take the
  sparse form on every row; every other tensor, all 31 040 one-hot rows of dense_2/kernel included, takes
  ApplyAdam's dense form.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import keras_eval
from . import ncf_train
from .ncf_train import as_dtype, epoch_orders  # noqa: F401  (epoch_orders: the trainer's row order)

TABLES = ("fm_movieId_embedding", "fm_userId_embedding", "fm_movieGenre1_embedding", "fm_userGenre1_embedding",
          "deep_movieId_embedding", "deep_userId_embedding")
NUMERIC_KEYS = ("movieAvgRating", "movieRatingCount", "movieRatingStddev", "releaseYear",
                "userAvgRating", "userRatingCount", "userRatingStddev")


class Adam(ncf_train.Adam):
    """Keras Adam over DeepFM's variables: `ncf_train.Adam`'s state, hyper-parameters and formulas, with the six
    tables of TABLES as the IndexedSlices (sparse-form) variables in place of NeuralCF's two."""

    TABLES = TABLES

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
            if k in self.TABLES:
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


class Rows:
    """The columns one DeepFM step reads: ids (int64 [B]; genre -1 = missing) and the 7 numerics (float32 [B, 7],
    NUMERIC_KEYS order, numeric_column's cast)."""

    def __init__(self, mid, uid, ig, ug, num, y=None):
        self.mid, self.uid, self.ig, self.ug = (np.asarray(a, np.int64) for a in (mid, uid, ig, ug))
        self.num = np.asarray(num, np.float32)
        self.y = None if y is None else np.asarray(y)

    @classmethod
    def from_features(cls, feats) -> "Rows":
        """From a feature dict whose movieGenre1 / userGenre1 are vocabulary indices (e.g. the golden npz files)."""
        num = np.stack([np.asarray(feats[k]).astype(np.float32) for k in NUMERIC_KEYS], axis=1)
        return cls(feats["movieId"], feats["userId"], feats["movieGenre1"], feats["userGenre1"], num,
                   feats.get("label"))

    def take(self, rows) -> "Rows":
        return Rows(self.mid[rows], self.uid[rows], self.ig[rows], self.ug[rows], self.num[rows],
                    None if self.y is None else self.y[rows])


def _lookup(table, ids, dtype):
    out = table.astype(dtype)[np.maximum(ids, 0)]
    out[ids < 0] = 0
    return out


def _sizes(W):
    G = W["fm_movieGenre1_embedding"].shape[0]
    Vm = W["fm_movieId_embedding"].shape[0]
    Vu = W["fm_userId_embedding"].shape[0]
    return G, Vm, Vu, 2 * G + Vm + Vu


def first_order_index(W, r: Rows):
    """[4][B] rows of dense_2/kernel the one-hots select (movieGenre1 | movieId | userGenre1 | userId), -1 for a
    missing genre."""
    G, Vm, _, _ = _sizes(W)
    return np.stack([np.where(r.ig >= 0, r.ig, -1), G + r.mid, np.where(r.ug >= 0, G + Vm + r.ug, -1),
                     2 * G + Vm + r.uid])


def forward(W, r: Rows, dtype=np.float32):
    """(p, z, cache): probabilities and logits [B] and what backward needs."""
    E = W["fm_movieId_embedding"].shape[1]
    _, _, _, fm1 = _sizes(W)
    item = _lookup(W["fm_movieId_embedding"], r.mid, dtype)
    user = _lookup(W["fm_userId_embedding"], r.uid, dtype)
    ig = _lookup(W["fm_movieGenre1_embedding"], r.ig, dtype)
    ug = _lookup(W["fm_userGenre1_embedding"], r.ug, dtype)
    dots = np.stack([np.sum(item * user, axis=1), np.sum(ig * ug, axis=1), np.sum(ig * user, axis=1),
                     np.sum(item * ug, axis=1)], axis=1).astype(dtype)
    num = r.num.astype(dtype)
    # sorted DenseFeatures concat: movieAvgRating | deep movieId | movieRatingCount, movieRatingStddev,
    # releaseYear, userAvgRating | deep userId | userRatingCount, userRatingStddev
    x = np.concatenate([num[:, 0:1], _lookup(W["deep_movieId_embedding"], r.mid, dtype), num[:, 1:5],
                        _lookup(W["deep_userId_embedding"], r.uid, dtype), num[:, 5:7]], axis=1)
    assert x.shape[1] == 7 + 2 * E
    a1 = x @ W["dense/kernel"].astype(dtype) + W["dense/bias"].reshape(-1).astype(dtype)
    h1 = np.maximum(a1, dtype(0))
    a2 = h1 @ W["dense_1/kernel"].astype(dtype) + W["dense_1/bias"].reshape(-1).astype(dtype)
    h2 = np.maximum(a2, dtype(0))
    K = W["dense_2/kernel"][:, 0].astype(dtype)
    fo = first_order_index(W, r)
    z = np.zeros(len(r.mid), dtype)
    for s in range(4):
        z = z + np.where(fo[s] >= 0, K[np.maximum(fo[s], 0)], dtype(0))
    z = (z + dots @ K[fm1:fm1 + 4] + h2 @ K[fm1 + 4:] + W["dense_2/bias"].reshape(-1)[0].astype(dtype)).astype(dtype)
    e = np.exp(-np.abs(z))                                     # stable sigmoid, both signs
    p = np.where(z >= 0, dtype(1) / (dtype(1) + e), e / (dtype(1) + e)).astype(dtype)
    return p, z, dict(item=item, user=user, ig=ig, ug=ug, dots=dots, x=x, h1=h1, h2=h2, fo=fo)


def batch_loss(W, r: Rows, y, dtype=np.float64) -> float:
    """Mean over the batch of max(z,0) - z*y + log1p(exp(-|z|))."""
    _, z, _ = forward(W, r, dtype)
    yv = np.asarray(y).astype(dtype)
    return float(np.mean(np.maximum(z, 0) - z * yv + np.log1p(np.exp(-np.abs(z)))))


def gradients(W, r: Rows, y, dtype=np.float32):
    """(grads, p, z): grads in the shapes of W.  Table gradients and the one-hot rows of dense_2/kernel are dense
    arrays that are zero off the batch; a repeated id sums its rows in row order (np.add.at)."""
    p, z, c = forward(W, r, dtype)
    B = len(r.mid)
    E = W["fm_movieId_embedding"].shape[1]
    _, _, _, fm1 = _sizes(W)
    dz = ((p - np.asarray(y).astype(dtype)) / dtype(B)).astype(dtype)
    K = W["dense_2/kernel"][:, 0].astype(dtype)
    g: Dict[str, np.ndarray] = {}
    gK = np.zeros(K.shape, dtype)
    for s in range(4):                                        # one-hot rows: dz at the selected rows
        ok = c["fo"][s] >= 0
        np.add.at(gK, c["fo"][s][ok], dz[ok])
    gK[fm1:fm1 + 4] = c["dots"].T @ dz
    gK[fm1 + 4:] = c["h2"].T @ dz
    g["dense_2/kernel"] = gK[:, None]
    g["dense_2/bias"] = np.array([dz.sum(dtype=dtype)], dtype)
    d2 = (dz[:, None] * K[None, fm1 + 4:]).astype(dtype) * (c["h2"] > 0)
    g["dense_1/kernel"] = (c["h1"].T @ d2).astype(dtype)
    g["dense_1/bias"] = d2.sum(0).astype(dtype)
    d1 = (d2 @ W["dense_1/kernel"].astype(dtype).T).astype(dtype) * (c["h1"] > 0)
    g["dense/kernel"] = (c["x"].T @ d1).astype(dtype)
    g["dense/bias"] = d1.sum(0).astype(dtype)
    dx = (d1 @ W["dense/kernel"].astype(dtype).T).astype(dtype)
    w0, w1, w2, w3 = (K[fm1 + d] for d in range(4))
    dzc = dz[:, None]
    parts = {
        "fm_movieId_embedding": (r.mid, dzc * (w0 * c["user"] + w3 * c["ug"])),
        "fm_userId_embedding": (r.uid, dzc * (w0 * c["item"] + w2 * c["ig"])),
        "fm_movieGenre1_embedding": (r.ig, dzc * (w1 * c["ug"] + w2 * c["user"])),
        "fm_userGenre1_embedding": (r.ug, dzc * (w1 * c["ig"] + w3 * c["item"])),
        "deep_movieId_embedding": (r.mid, dx[:, 1:1 + E]),
        "deep_userId_embedding": (r.uid, dx[:, 5 + E:5 + 2 * E]),
    }
    for name, (ids, part) in parts.items():
        G = np.zeros(W[name].shape, dtype)
        ok = ids >= 0                                          # a missing genre gives no entry
        np.add.at(G, ids[ok], part[ok].astype(dtype))
        g[name] = G
    return g, p, z


def table_rows(r: Rows) -> Dict[str, np.ndarray]:
    """The batch's rows of each table (lazy Adam only)."""
    return {"fm_movieId_embedding": r.mid, "fm_userId_embedding": r.uid,
            "fm_movieGenre1_embedding": r.ig[r.ig >= 0], "fm_userGenre1_embedding": r.ug[r.ug >= 0],
            "deep_movieId_embedding": r.mid, "deep_userId_embedding": r.uid}


def fit(W, data: Rows, label, orders, batch_size: int, dtype=np.float32, hp=None, lazy: bool = False,
        max_steps: Optional[int] = None, keep_outputs: bool = False):
    """`model.fit` over the rows in `orders` [epochs][n], batches of `batch_size` consecutive entries, the last one
    partial; as `ncf_train.fit`.  Returns (weights at `dtype`, history, outputs, Adam)."""
    W = as_dtype(W, dtype)
    opt = Adam(W, dtype, hp, lazy)
    label = np.asarray(label)
    history: List[dict] = []
    outputs = [] if keep_outputs else None
    steps = 0
    for order in orders:
        ps, zs, ys = [], [], []
        for lo in range(0, len(order), batch_size):
            if max_steps is not None and steps >= max_steps:
                break
            rows = np.asarray(order[lo:lo + batch_size])
            r, y = data.take(rows), label[rows]
            g, p, z = gradients(W, r, y, dtype)
            opt.step(W, g, table_rows(r))
            ps.append(p); zs.append(z); ys.append(y)
            if keep_outputs:
                outputs.append((p.copy(), z.copy(), y.copy()))
            steps += 1
        if ps:
            res = keras_eval.keras_evaluate(np.concatenate(ps).astype(np.float32),
                                            np.concatenate(zs).astype(np.float32), np.concatenate(ys))
            history.append({k: res[k] for k in ("loss", "accuracy", "roc_auc", "pr_auc")})
        if max_steps is not None and steps >= max_steps:
            break
    return W, history, outputs, opt
