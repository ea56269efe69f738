"""CPU oracle of `model.fit` for Wide&Deep, the training call of the reference's WideNDeep.py:
`compile(loss='binary_crossentropy', optimizer='adam', ...)` and `fit(train_dataset, epochs=5)`.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

What one step computes (DESIGN.md section 4.18), in numpy at `dtype` (float32 or float64), statement by statement
like oracle/deepfm_train.py:

* forward: `ctr_oracle.widendeep_forward` - the deep input is DenseFeatures' sorted concat of the 7 numerics and
  the ten embedding columns (movieGenre1..3, movieId, userGenre1..5, userId; a missing or out-of-vocabulary genre,
  index -1, is a zero row), through Dense(relu) -> Dense(relu); dense_2 over [deep | one-hot of
  crossed_column(movieId, userRatedMovie1)] -> logit z, p = sigmoid(z);
* loss: the logit-path binary cross-entropy, mean over the batch, so dL/dz_i = (p_i - y_i) / B_batch;
* backward: dense_2's deep rows get dz . h2, its wide row at the row's crossed bucket gets dz (rows sharing a
  bucket add up); the MLP with relu' = [a > 0] into dense_1, dense and the ten embedding slots.  A missing genre
  gives no entry (safe_embedding_lookup_sparse prunes it); an id that repeats within a batch gets the sum of its
  rows' gradients, in row order;
* Keras Adam (`Adam`, `ncf_train.Adam`'s state and formulas): the ten tables take the sparse form on every row;
  every Dense tensor, all `cross_buckets` wide rows of dense_2/kernel included, takes ApplyAdam's dense form.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import ctr_oracle, deepfm_train, keras_eval
from .ncf_train import as_dtype, epoch_orders  # noqa: F401  (epoch_orders: the trainer's row order)

MOVIE_GENRES = tuple("movieGenre%d_embedding" % k for k in (1, 2, 3))
USER_GENRES = tuple("userGenre%d_embedding" % k for k in (1, 2, 3, 4, 5))
TABLES = MOVIE_GENRES + ("movieId_embedding",) + USER_GENRES + ("userId_embedding",)   # the kernel's slot order
NUMERIC_KEYS = deepfm_train.NUMERIC_KEYS


class Adam(deepfm_train.Adam):
    """Keras Adam over Wide&Deep's variables: `ncf_train.Adam`'s state, hyper-parameters and formulas, with the ten
    tables of TABLES as the IndexedSlices (sparse-form) variables."""

    TABLES = TABLES


class Rows:
    """The columns one Wide&Deep step reads: movieId, userId, userRatedMovie1 (int64 [B]), the genre indices
    (int64 [B, 3] and [B, 5]; -1 = missing) and the 7 numerics (float32 [B, 7], NUMERIC_KEYS order)."""

    def __init__(self, mid, uid, mg, ug, num, rated, y=None):
        self.mid, self.uid, self.rated = (np.asarray(a, np.int64) for a in (mid, uid, rated))
        self.mg = np.asarray(mg, np.int64).reshape(len(self.mid), 3)
        self.ug = np.asarray(ug, np.int64).reshape(len(self.mid), 5)
        self.num = np.asarray(num, np.float32)
        self.y = None if y is None else np.asarray(y)
        self._buckets: Dict[int, np.ndarray] = {}

    @classmethod
    def from_features(cls, feats) -> "Rows":
        """From a feature dict whose genre columns are vocabulary indices (e.g. the golden npz files)."""
        num = np.stack([np.asarray(feats[k]).astype(np.float32) for k in NUMERIC_KEYS], axis=1)
        mg = np.stack([np.asarray(feats["movieGenre%d" % k]) for k in (1, 2, 3)], axis=1)
        ug = np.stack([np.asarray(feats["userGenre%d" % k]) for k in (1, 2, 3, 4, 5)], axis=1)
        return cls(feats["movieId"], feats["userId"], mg, ug, num, feats["userRatedMovie1"], feats.get("label"))

    def bucket(self, cross_buckets: int) -> np.ndarray:
        """Each row's crossed_column(movieId, userRatedMovie1) bucket (computed once per size)."""
        if cross_buckets not in self._buckets:
            self._buckets[cross_buckets] = ctr_oracle.crossed_bucket_array(self.mid, self.rated, cross_buckets)
        return self._buckets[cross_buckets]

    def take(self, rows) -> "Rows":
        r = Rows(self.mid[rows], self.uid[rows], self.mg[rows], self.ug[rows], self.num[rows], self.rated[rows],
                 None if self.y is None else self.y[rows])
        r._buckets = {k: v[rows] for k, v in self._buckets.items()}
        return r

    def ids(self) -> List[np.ndarray]:
        """The ten slots' ids [B] in TABLES order."""
        return [self.mg[:, 0], self.mg[:, 1], self.mg[:, 2], self.mid] + [self.ug[:, k] for k in range(5)] + \
            [self.uid]

    def features(self) -> dict:
        """The feature dict of these rows (genres as indices), as `ctr_oracle` and the library take it."""
        f = {"movieId": self.mid, "userId": self.uid, "userRatedMovie1": self.rated}
        f.update({"movieGenre%d" % (k + 1): self.mg[:, k] for k in range(3)})
        f.update({"userGenre%d" % (k + 1): self.ug[:, k] for k in range(5)})
        f.update({k: self.num[:, j] for j, k in enumerate(NUMERIC_KEYS)})
        if self.y is not None:
            f["label"] = self.y
        return f


def _lookup(table, ids, dtype):
    out = table.astype(dtype)[np.maximum(ids, 0)]
    out[ids < 0] = 0
    return out


def slot_columns(E: int) -> List[int]:
    """The first row of dense/kernel of each slot (TABLES order) in DenseFeatures' sorted concat: movieAvgRating |
    movieGenre1..3 | movieId | 4 numerics | userGenre1..5 | userId | 2 numerics."""
    return [1, 1 + E, 1 + 2 * E, 1 + 3 * E] + [5 + 4 * E + k * E for k in range(5)] + [5 + 9 * E]


def cross_buckets(W) -> int:
    return W["dense_2/kernel"].shape[0] - W["dense_1/kernel"].shape[1]


def forward(W, r: Rows, dtype=np.float32):
    """(p, z, cache): probabilities and logits [B] and what backward needs."""
    E = W["movieId_embedding"].shape[1]
    num = r.num.astype(dtype)
    e = [_lookup(W[name], ids, dtype) for name, ids in zip(TABLES, r.ids())]
    x = np.concatenate([num[:, 0:1], e[0], e[1], e[2], e[3], num[:, 1:5], *e[4:9], e[9], num[:, 5:7]], axis=1)
    assert x.shape[1] == 7 + 10 * E
    a1 = x @ W["dense/kernel"].astype(dtype) + W["dense/bias"].reshape(-1).astype(dtype)
    h1 = np.maximum(a1, dtype(0))
    a2 = h1 @ W["dense_1/kernel"].astype(dtype) + W["dense_1/bias"].reshape(-1).astype(dtype)
    h2 = np.maximum(a2, dtype(0))
    K = W["dense_2/kernel"][:, 0].astype(dtype)
    hw = h2.shape[1]
    bucket = r.bucket(cross_buckets(W))
    z = (h2 @ K[:hw] + K[hw + bucket] + W["dense_2/bias"].reshape(-1)[0].astype(dtype)).astype(dtype)
    ez = np.exp(-np.abs(z))                                    # stable sigmoid, both signs
    p = np.where(z >= 0, dtype(1) / (dtype(1) + ez), ez / (dtype(1) + ez)).astype(dtype)
    return p, z, dict(x=x, h1=h1, h2=h2, bucket=bucket)


def batch_loss(W, r: Rows, y, dtype=np.float64) -> float:
    """Mean over the batch of max(z,0) - z*y + log1p(exp(-|z|))."""
    _, z, _ = forward(W, r, dtype)
    yv = np.asarray(y).astype(dtype)
    return float(np.mean(np.maximum(z, 0) - z * yv + np.log1p(np.exp(-np.abs(z)))))


def gradients(W, r: Rows, y, dtype=np.float32):
    """(grads, p, z): grads in the shapes of W.  Table gradients and the wide rows of dense_2/kernel are dense
    arrays that are zero off the batch; a repeated id or bucket sums its rows in row order (np.add.at)."""
    p, z, c = forward(W, r, dtype)
    B = len(r.mid)
    E = W["movieId_embedding"].shape[1]
    dz = ((p - np.asarray(y).astype(dtype)) / dtype(B)).astype(dtype)
    K = W["dense_2/kernel"][:, 0].astype(dtype)
    hw = c["h2"].shape[1]
    g: Dict[str, np.ndarray] = {}
    gK = np.zeros(K.shape, dtype)
    gK[:hw] = c["h2"].T @ dz
    np.add.at(gK, hw + c["bucket"], dz)                        # the wide rows: dz at each row's bucket
    g["dense_2/kernel"] = gK[:, None]
    g["dense_2/bias"] = np.array([dz.sum(dtype=dtype)], dtype)
    d2 = (dz[:, None] * K[None, :hw]).astype(dtype) * (c["h2"] > 0)
    g["dense_1/kernel"] = (c["h1"].T @ d2).astype(dtype)
    g["dense_1/bias"] = d2.sum(0).astype(dtype)
    d1 = (d2 @ W["dense_1/kernel"].astype(dtype).T).astype(dtype) * (c["h1"] > 0)
    g["dense/kernel"] = (c["x"].T @ d1).astype(dtype)
    g["dense/bias"] = d1.sum(0).astype(dtype)
    dx = (d1 @ W["dense/kernel"].astype(dtype).T).astype(dtype)
    for name, ids, col in zip(TABLES, r.ids(), slot_columns(E)):
        G = np.zeros(W[name].shape, dtype)
        ok = ids >= 0                                          # a missing genre gives no entry
        np.add.at(G, ids[ok], dx[ok, col:col + E])
        g[name] = G
    return g, p, z


def table_rows(r: Rows) -> Dict[str, np.ndarray]:
    """The batch's rows of each table (lazy Adam only)."""
    return {name: ids[ids >= 0] for name, ids in zip(TABLES, r.ids())}


def fit(W, data: Rows, label, orders, batch_size: int, dtype=np.float32, hp=None, lazy: bool = False,
        max_steps: Optional[int] = None, keep_outputs: bool = False):
    """`model.fit` over the rows in `orders` [epochs][n], batches of `batch_size` consecutive entries, the last one
    partial; as `deepfm_train.fit`.  Returns (weights at `dtype`, history, outputs, Adam)."""
    W = as_dtype(W, dtype)
    opt = Adam(W, dtype, hp, lazy)
    label = np.asarray(label)
    data.bucket(cross_buckets(W))                              # once for all the rows
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


def fit_validate(W, features, orders, batch_size: int, dtype=np.float32, val=None, validation_freq: int = 1, opt=None,
                 hp=None):
    """`model.fit(..., validation_data=val, validation_freq=...)` over the rows of the feature dict `features`
    (labels in "label"), as `oracle.fit_validation.fit` states it for NeuralCF and DeepFM: after every epoch e with
    (e + 1) % validation_freq == 0, `keras_evaluate` of the forward of `val` at `dtype`.  `opt`: the Adam state of an
    earlier call to continue from.  Returns (weights at `dtype`, history, val_history, Adam); val_history holds None
    for the epochs not validated.  Epoch by epoch, continuing with `opt`, gives the bits of one call."""
    metrics = ("loss", "accuracy", "roc_auc", "pr_auc")

    def summary(p, z, y):
        r = keras_eval.keras_evaluate(np.asarray(p).astype(np.float32), np.asarray(z).astype(np.float32),
                                      np.asarray(y))
        return {k: r[k] for k in metrics}

    rows = Rows.from_features(features)
    label = np.asarray(features["label"])
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
