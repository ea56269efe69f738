"""CPU oracle of `model.fit` for DeepFM_v2, the training call of the reference's DeepFM_v2.py:
`compile(loss='binary_crossentropy', optimizer='adam', ...)` and `fit(train_dataset, epochs=5)`.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

What one step computes (DESIGN.md section 4.19), in numpy at `dtype` (float32 or float64), statement by statement
like oracle/deepfm_train.py:

* forward: `ctr_oracle.deepfm_v2_forward` - first = the four one-hot weights of first_cat/kernel (movieGenre1 |
  movieId | userGenre1 | userId; none for a missing genre, index -1) + first_cat/bias + first_num(numerics); the
  five fields F_f = proj_f(x_f) (the four embedding rows, a missing genre a zero row, and the raw numerics); the
  deep MLP over Flatten(F) through Dense(relu) -> Dense(relu); fm_c = (sum_f F_fc)^2 - sum_f F_fc^2 (no 1/2);
  out over [first | fm | deep] -> logit z, p = sigmoid(z);
* loss: the logit-path binary cross-entropy, mean over the batch, so dL/dz_i = (p_i - y_i) / B_batch;
* backward: out/kernel gets [first | fm | deep] . dz; dfirst = dz * out/kernel[0] goes to first_cat/bias,
  first_num/bias, first_num/kernel (times the numerics) and the four selected one-hot rows of first_cat/kernel;
  dF_fc = dz * out/kernel[1 + c] * 2 (s_c - F_fc) plus deep/kernel . delta1 of the MLP (relu' = [a > 0]); then
  proj_f/kernel gets x_f (x) dF_f, proj_f/bias dF_f (a row whose genre is missing too: its input is a zero vector)
  and the table row proj_f/kernel . dF_f (none for a missing genre).  An id that repeats within a batch gets the
  sum of its rows' gradients, in row order;
* Keras Adam (`Adam`, `deepfm_train.Adam`'s state and formulas): the four tables take the sparse form on every row;
  every other tensor, all fm1_width one-hot rows of first_cat/kernel included, takes ApplyAdam's dense form.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import deepfm_train, keras_eval
from .ncf_train import as_dtype, epoch_orders  # noqa: F401  (epoch_orders: the trainer's row order)

TABLES = ("movieGenre1_embedding", "movieId_embedding", "userGenre1_embedding", "userId_embedding")   # field order
FIELDS = ("movieGenre1", "movieId", "userGenre1", "userId")
NUMERIC_KEYS = deepfm_train.NUMERIC_KEYS
Rows = deepfm_train.Rows          # the same columns as DeepFM: movieId, userId, movieGenre1, userGenre1, numerics


class Adam(deepfm_train.Adam):
    """Keras Adam over DeepFM_v2's variables: `deepfm_train.Adam`'s state, hyper-parameters and formulas, with the
    four tables of TABLES as the IndexedSlices (sparse-form) variables."""

    TABLES = TABLES


def features(r: Rows) -> dict:
    """The feature dict of rows r (genres as indices), as `ctr_oracle` and the library take it."""
    f = {"movieId": r.mid, "userId": r.uid, "movieGenre1": r.ig, "userGenre1": r.ug}
    f.update({k: r.num[:, j] for j, k in enumerate(NUMERIC_KEYS)})
    if r.y is not None:
        f["label"] = r.y
    return f


def _lookup(table, ids, dtype):
    out = table.astype(dtype)[np.maximum(ids, 0)]
    out[ids < 0] = 0
    return out


def _ids(r: Rows):
    return [r.ig, r.mid, r.ug, r.uid]


def first_order_index(W, r: Rows):
    """[4][B] rows of first_cat/kernel the one-hots select (movieGenre1 | movieId | userGenre1 | userId), -1 for a
    missing genre."""
    G = W["movieGenre1_embedding"].shape[0]
    Vm = W["movieId_embedding"].shape[0]
    return np.stack([np.where(r.ig >= 0, r.ig, -1), G + r.mid, np.where(r.ug >= 0, G + Vm + r.ug, -1),
                     2 * G + Vm + r.uid])


def forward(W, r: Rows, dtype=np.float32):
    """(p, z, cache): probabilities and logits [B] and what backward needs."""
    num = r.num.astype(dtype)
    B = len(r.mid)
    K1 = W["first_cat/kernel"][:, 0].astype(dtype)
    fo = first_order_index(W, r)
    first = np.zeros(B, dtype)
    for s in range(4):
        first = first + np.where(fo[s] >= 0, K1[np.maximum(fo[s], 0)], dtype(0))
    first = first + W["first_cat/bias"].reshape(-1)[0].astype(dtype)
    first = (first + (num @ W["first_num/kernel"][:, 0].astype(dtype) +
                      W["first_num/bias"].reshape(-1)[0].astype(dtype))).astype(dtype)
    x = [_lookup(W[t], ids, dtype) for t, ids in zip(TABLES, _ids(r))]
    F = [x[f] @ W["proj_%s/kernel" % FIELDS[f]].astype(dtype) + W["proj_%s/bias" % FIELDS[f]].astype(dtype)
         for f in range(4)]
    F.append(num @ W["proj_num/kernel"].astype(dtype) + W["proj_num/bias"].astype(dtype))
    F = np.stack(F, axis=1).astype(dtype)                      # [B, 5, P]
    flat = F.reshape(B, -1)
    a1 = flat @ W["deep/kernel"].astype(dtype) + W["deep/bias"].astype(dtype)
    h1 = np.maximum(a1, dtype(0))
    a2 = h1 @ W["deep_1/kernel"].astype(dtype) + W["deep_1/bias"].astype(dtype)
    h2 = np.maximum(a2, dtype(0))
    s = F.sum(axis=1)
    fm = (s * s - (F * F).sum(axis=1)).astype(dtype)          # no 1/2 (DeepFM_v2.py:147-152)
    Ko = W["out/kernel"][:, 0].astype(dtype)
    P = F.shape[2]
    z = (first * Ko[0] + fm @ Ko[1:1 + P] + h2 @ Ko[1 + P:] + W["out/bias"].reshape(-1)[0].astype(dtype)).astype(dtype)
    e = np.exp(-np.abs(z))                                     # stable sigmoid, both signs
    p = np.where(z >= 0, dtype(1) / (dtype(1) + e), e / (dtype(1) + e)).astype(dtype)
    return p, z, dict(num=num, x=x, first=first, F=F, s=s, fm=fm, h1=h1, h2=h2, fo=fo)


def batch_loss(W, r: Rows, y, dtype=np.float64) -> float:
    """Mean over the batch of max(z,0) - z*y + log1p(exp(-|z|))."""
    _, z, _ = forward(W, r, dtype)
    yv = np.asarray(y).astype(dtype)
    return float(np.mean(np.maximum(z, 0) - z * yv + np.log1p(np.exp(-np.abs(z)))))


def gradients(W, r: Rows, y, dtype=np.float32, fm_half: bool = False):
    """(grads, p, z): grads in the shapes of W.  Table gradients and the one-hot rows of first_cat/kernel are dense
    arrays that are zero off the batch; a repeated id sums its rows in row order (np.add.at).  `fm_half` (a mutant
    for the tests): the FM gradient of the textbook 1/2 (s_c - F_fc) instead of the script's 2 (s_c - F_fc)."""
    p, z, c = forward(W, r, dtype)
    B = len(r.mid)
    F = c["F"]
    P = F.shape[2]
    dz = ((p - np.asarray(y).astype(dtype)) / dtype(B)).astype(dtype)
    Ko = W["out/kernel"][:, 0].astype(dtype)
    g: Dict[str, np.ndarray] = {}
    g["out/kernel"] = np.concatenate([[c["first"] @ dz], c["fm"].T @ dz, c["h2"].T @ dz]).astype(dtype)[:, None]
    g["out/bias"] = np.array([dz.sum(dtype=dtype)], dtype)
    dfirst = (dz * Ko[0]).astype(dtype)
    gK1 = np.zeros(W["first_cat/kernel"].shape[0], dtype)
    for s in range(4):                                         # one-hot rows: dfirst at the selected rows
        ok = c["fo"][s] >= 0
        np.add.at(gK1, c["fo"][s][ok], dfirst[ok])
    g["first_cat/kernel"] = gK1[:, None]
    g["first_cat/bias"] = np.array([dfirst.sum(dtype=dtype)], dtype)
    g["first_num/kernel"] = (c["num"].T @ dfirst).astype(dtype)[:, None]
    g["first_num/bias"] = np.array([dfirst.sum(dtype=dtype)], dtype)
    d2 = (dz[:, None] * Ko[None, 1 + P:]).astype(dtype) * (c["h2"] > 0)
    g["deep_1/kernel"] = (c["h1"].T @ d2).astype(dtype)
    g["deep_1/bias"] = d2.sum(0).astype(dtype)
    d1 = (d2 @ W["deep_1/kernel"].astype(dtype).T).astype(dtype) * (c["h1"] > 0)
    g["deep/kernel"] = (F.reshape(B, -1).T @ d1).astype(dtype)
    g["deep/bias"] = d1.sum(0).astype(dtype)
    dF = (d1 @ W["deep/kernel"].astype(dtype).T).astype(dtype).reshape(F.shape)
    k = dtype(0.5) if fm_half else dtype(2)
    dF = (dF + (dz[:, None] * Ko[None, 1:1 + P])[:, None, :] * k * (c["s"][:, None, :] - F)).astype(dtype)
    for f in range(4):
        name = FIELDS[f]
        g["proj_%s/kernel" % name] = (c["x"][f].T @ dF[:, f]).astype(dtype)
        g["proj_%s/bias" % name] = dF[:, f].sum(0).astype(dtype)   # a missing genre's row included
        dx = (dF[:, f] @ W["proj_%s/kernel" % name].astype(dtype).T).astype(dtype)
        ids = _ids(r)[f]
        G = np.zeros(W[TABLES[f]].shape, dtype)
        ok = ids >= 0                                          # a missing genre gives no entry
        np.add.at(G, ids[ok], dx[ok])
        g[TABLES[f]] = G
    g["proj_num/kernel"] = (c["num"].T @ dF[:, 4]).astype(dtype)
    g["proj_num/bias"] = dF[:, 4].sum(0).astype(dtype)
    return g, p, z


def table_rows(r: Rows) -> Dict[str, np.ndarray]:
    """The batch's rows of each table (lazy Adam only)."""
    return {"movieGenre1_embedding": r.ig[r.ig >= 0], "movieId_embedding": r.mid,
            "userGenre1_embedding": r.ug[r.ug >= 0], "userId_embedding": r.uid}


def fit(W, data: Rows, label, orders, batch_size: int, dtype=np.float32, hp=None, lazy: bool = False,
        max_steps: Optional[int] = None, keep_outputs: bool = False):
    """`model.fit` over the rows in `orders` [epochs][n], batches of `batch_size` consecutive entries, the last one
    partial; as `deepfm_train.fit`.  Returns (weights at `dtype`, history, outputs, Adam)."""
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


def fit_validate(W, feats, orders, batch_size: int, dtype=np.float32, val=None, validation_freq: int = 1, opt=None,
                 hp=None):
    """`model.fit(..., validation_data=val, validation_freq=...)` over the rows of the feature dict `feats` (labels
    in "label"), as `oracle.fit_validation.fit` states it for NeuralCF and DeepFM: after every epoch e with
    (e + 1) % validation_freq == 0, `keras_evaluate` of the forward of `val` at `dtype`.  `opt`: the Adam state of an
    earlier call to continue from.  Returns (weights at `dtype`, history, val_history, Adam); val_history holds None
    for the epochs not validated.  Epoch by epoch, continuing with `opt`, gives the bits of one call."""
    metrics = ("loss", "accuracy", "roc_auc", "pr_auc")

    def summary(p, z, y):
        r = keras_eval.keras_evaluate(np.asarray(p).astype(np.float32), np.asarray(z).astype(np.float32),
                                      np.asarray(y))
        return {k: r[k] for k in metrics}

    rows = Rows.from_features(feats)
    label = np.asarray(feats["label"])
    W = as_dtype(W, dtype)
    if opt is None:
        opt = Adam(W, dtype, hp)
    vrows = None if val is None else Rows.from_features(val)
    history: List[dict] = []
    val_history: List[Optional[dict]] = []
    for e, order in enumerate(orders):
        ps, zs, ys = [], [], []
        for lo in range(0, len(order), batch_size):
            idx = np.asarray(order[lo:lo + batch_size])
            r, y = rows.take(idx), label[idx]
            g, p, z = gradients(W, r, y, dtype)
            opt.step(W, g, table_rows(r))
            ps.append(p); zs.append(z); ys.append(y)
        history.append(summary(np.concatenate(ps), np.concatenate(zs), np.concatenate(ys)))
        if vrows is not None and (e + 1) % validation_freq == 0:
            p, z, _ = forward(W, vrows, dtype)
            val_history.append(summary(p, z, val["label"]))
        else:
            val_history.append(None)
    return W, history, val_history, opt
