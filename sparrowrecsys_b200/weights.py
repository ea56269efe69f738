"""Weight inventory and initialisers of the reference CTR graphs.

Canonical tensor names and shapes per model (SURVEY.md appendix A).  Shapes are
the *reference's* (Keras/TF variable shapes: Dense kernel `[in, out]`, embedding
tables `[buckets, E]`); the device re-layout (row padding, column permutation,
hi/lo splits) is private to the CUDA library and happens in `srs_model_create`.

`init_weights` draws from the reference's own initialisers (SURVEY.md section 8a):
`embedding_column` -> truncated_normal(stddev=1/sqrt(E)); `Embedding` layer ->
uniform(-0.05, 0.05); Dense kernel -> glorot_uniform, bias -> 0; PReLU alpha ->
0.  With `for_test=True` biases/alphas are made non-zero and the Dense rows that
multiply raw-scale numerics (releaseYear ~ 1990, movieRatingCount up to 14616)
are rescaled so logits stay O(1) -- otherwise sigmoid saturates and a 1e-4 check
on probabilities is vacuous (SURVEY.md section 8c "residual risk").
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from .spec import ModelSpec

# typical magnitude of each numeric column in NUMERIC_KEYS order
# (movieAvgRating, movieRatingCount, movieRatingStddev, releaseYear,
#  userAvgRating, userRatingCount, userRatingStddev)
_NUMERIC_SCALE = np.array([4.0, 8000.0, 1.5, 2000.0, 4.0, 60.0, 2.0], dtype=np.float32)


def weight_shapes(spec: ModelSpec) -> List[Tuple[str, Tuple[int, ...]]]:
    E, Vm, Vu, G = spec.emb_dim, spec.n_movies, spec.n_users, spec.n_genres
    h = spec.hidden
    m = spec.model
    out: List[Tuple[str, Tuple[int, ...]]] = []
    add = lambda n, *s: out.append((n, tuple(s)))
    if m in ("embeddingmlp", "widendeep"):
        for k in range(1, 4):
            add("movieGenre%d_embedding" % k, G, E)
        for k in range(1, 6):
            add("userGenre%d_embedding" % k, G, E)
        add("movieId_embedding", Vm, E)
        add("userId_embedding", Vu, E)
        add("dense/kernel", 7 + 10 * E, h[0]); add("dense/bias", h[0])
        add("dense_1/kernel", h[0], h[1]); add("dense_1/bias", h[1])
        last_in = h[1] + (spec.cross_buckets if m == "widendeep" else 0)
        add("dense_2/kernel", last_in, 1); add("dense_2/bias", 1)
    elif m == "neuralcf":
        add("movieId_embedding", Vm, E)
        add("userId_embedding", Vu, E)
        dims = [2 * E, *h, 1]
        for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
            add("dense_%d/kernel" % i, a, b); add("dense_%d/bias" % i, b)
    elif m == "twotowers":
        add("movieId_embedding", Vm, E)
        add("userId_embedding", Vu, E)
        dims = [E, *h]
        for side in ("item", "user"):
            for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
                add("%s_dense_%d/kernel" % (side, i), a, b)
                add("%s_dense_%d/bias" % (side, i), b)
        if spec.final_dense:
            add("dense_out/kernel", 1, 1); add("dense_out/bias", 1)
    elif m == "deepfm":
        add("fm_movieId_embedding", Vm, E)
        add("fm_userId_embedding", Vu, E)
        add("fm_movieGenre1_embedding", G, E)
        add("fm_userGenre1_embedding", G, E)
        add("deep_movieId_embedding", Vm, E)
        add("deep_userId_embedding", Vu, E)
        add("dense/kernel", 7 + 2 * E, h[0]); add("dense/bias", h[0])
        add("dense_1/kernel", h[0], h[1]); add("dense_1/bias", h[1])
        add("dense_2/kernel", spec.fm1_width + 4 + h[1], 1); add("dense_2/bias", 1)
    elif m == "deepfm_v2":
        P = spec.proj_dim
        add("movieGenre1_embedding", G, E)
        add("movieId_embedding", Vm, E)
        add("userGenre1_embedding", G, E)
        add("userId_embedding", Vu, E)
        add("first_cat/kernel", spec.fm1_width, 1); add("first_cat/bias", 1)
        add("first_num/kernel", 7, 1); add("first_num/bias", 1)
        for f in ("movieGenre1", "movieId", "userGenre1", "userId"):
            add("proj_%s/kernel" % f, E, P); add("proj_%s/bias" % f, P)
        add("proj_num/kernel", 7, P); add("proj_num/bias", P)
        add("deep/kernel", 5 * P, h[0]); add("deep/bias", h[0])
        add("deep_1/kernel", h[0], h[1]); add("deep_1/bias", h[1])
        add("out/kernel", 1 + P + h[1], 1); add("out/bias", 1)
    elif m == "din":
        T, A = spec.hist_len, spec.au_hidden
        add("embedding", Vm, E)                 # Keras Embedding shared by candidate + history
        add("userId_embedding", Vu, E)
        add("userGenre1_embedding", G, E)
        add("movieGenre1_embedding", G, E)
        add("au_dense/kernel", 4 * E, A); add("au_dense/bias", A)
        add("au_prelu/alpha", T, A)
        add("au_out/kernel", A, 1); add("au_out/bias", 1)
        add("dense/kernel", 5 * E + 7, h[0]); add("dense/bias", h[0])
        add("prelu/alpha", h[0])
        add("dense_1/kernel", h[0], h[1]); add("dense_1/bias", h[1])
        add("prelu_1/alpha", h[1])
        add("dense_2/kernel", h[1], 1); add("dense_2/bias", 1)
    elif m == "dien":
        A = spec.au_hidden
        add("embedding", Vm, E)                 # DIEN.py:161 shared by candidate + history
        add("userId_embedding", Vu, E)
        add("userGenre1_embedding", G, E)
        add("movieGenre1_embedding", G, E)
        # tf.keras.layers.GRU(E) (DIEN.py:169): gates z | r | h, reset_after=True -> bias [2,3E]
        add("gru/kernel", E, 3 * E); add("gru_recurrent/kernel", E, 3 * E); add("gru/bias", 2, 3 * E)
        add("att_dense/kernel", E, A); add("att_dense/bias", A)        # DIEN.py:178
        add("att_out/kernel", A, 1); add("att_out/bias", 1)           # DIEN.py:179
        for g in ("r", "z", "h"):               # GRU_gate_parameter x3 (DIEN.py:204-219,229-232)
            add("augru_%s_input/kernel" % g, E, E); add("augru_%s_input/bias" % g, E)
            add("augru_%s_hidden/kernel" % g, E, E)
            add("augru_%s_act/kernel" % g, E, E); add("augru_%s_act/bias" % g, E)
        add("augru_h0", 1, E)                   # the stored initial state (see oracle dien_forward)
        add("dense/kernel", 5 * E + 7, h[0]); add("dense/bias", h[0])
        add("prelu/alpha", h[0])
        add("dense_1/kernel", h[0], h[1]); add("dense_1/bias", h[1])
        add("prelu_1/alpha", h[1])
        add("dense_2/kernel", h[1], 1); add("dense_2/bias", 1)
    else:
        raise AssertionError(m)
    return out


def _glorot(rng, fan_in, fan_out, shape):
    lim = np.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-lim, lim, size=shape).astype(np.float32)


def _trunc_normal(rng, shape, std):
    x = rng.standard_normal(size=shape)
    bad = np.abs(x) > 2.0
    while bad.any():                       # TF truncated_normal re-draws beyond 2 sigma
        x[bad] = rng.standard_normal(size=int(bad.sum()))
        bad = np.abs(x) > 2.0
    return (x * std).astype(np.float32)


def numeric_rows(spec: ModelSpec) -> Dict[str, np.ndarray]:
    """For each first Dense kernel that sees raw numerics: the kernel row index of
    each numeric in NUMERIC_KEYS order (rows follow DenseFeatures' sorted concat)."""
    E = spec.emb_dim
    m = spec.model
    if m in ("embeddingmlp", "widendeep"):
        # sorted: movieAvgRating, mG1..3_emb, movieId_emb, movieRatingCount,
        # movieRatingStddev, releaseYear, userAvgRating, uG1..5_emb, userId_emb,
        # userRatingCount, userRatingStddev
        return {"dense/kernel": np.array([0, 1 + 4 * E, 2 + 4 * E, 3 + 4 * E, 4 + 4 * E,
                                          5 + 10 * E, 6 + 10 * E])}
    if m == "deepfm":
        # sorted: movieAvgRating, movieId_emb, movieRatingCount, movieRatingStddev,
        # releaseYear, userAvgRating, userId_emb, userRatingCount, userRatingStddev
        return {"dense/kernel": np.array([0, 1 + E, 2 + E, 3 + E, 4 + E, 5 + 2 * E, 6 + 2 * E])}
    if m == "deepfm_v2":
        r = np.arange(7)
        return {"first_num/kernel": r, "proj_num/kernel": r}
    if m == "din":
        # [user_profile | pooled | candidate | context]
        # user_profile sorted: userAvgRating, userGenre1_emb, userId_emb, userRatingCount,
        #                      userRatingStddev
        # context sorted: movieAvgRating, movieGenre1_emb, movieRatingCount,
        #                 movieRatingStddev, releaseYear
        up = 0
        ctx = 2 * E + 3 + 2 * E
        return {"dense/kernel": np.array([ctx + 0, ctx + 1 + E, ctx + 2 + E, ctx + 3 + E,
                                          up + 0, up + 1 + 2 * E, up + 2 + 2 * E])}
    if m == "dien":
        # [augru | candidate | user_profile | context] (DIEN.py:250), blocks sorted as in DIN
        up = 2 * E
        ctx = 4 * E + 3
        return {"dense/kernel": np.array([ctx + 0, ctx + 1 + E, ctx + 2 + E, ctx + 3 + E,
                                          up + 0, up + 1 + 2 * E, up + 2 + 2 * E])}
    return {}


def init_weights(spec: ModelSpec, seed: int = 0, *, for_test: bool = True,
                 skip: Tuple[str, ...] = ()) -> Dict[str, np.ndarray]:
    """Seeded weights with the reference's initialisers.  `skip` names tensors to
    leave out (e.g. a 25.6 GB table that is generated on the device instead)."""
    rng = np.random.default_rng(seed)
    E = spec.emb_dim
    W: Dict[str, np.ndarray] = {}
    for name, shape in weight_shapes(spec):
        if name in skip:
            continue
        if name == "embedding":                       # tf.keras.layers.Embedding
            W[name] = rng.uniform(-0.05, 0.05, size=shape).astype(np.float32)
        elif name.endswith("_embedding"):             # feature_column.embedding_column
            W[name] = _trunc_normal(rng, shape, 1.0 / np.sqrt(E))
        elif name == "augru_h0":                      # GlorotUniform()(shape=(1, E)), DIEN.py:235-236
            W[name] = _glorot(rng, 1, E, shape)
        elif name.endswith("/kernel"):                # (Keras draws the GRU recurrent kernel
            W[name] = _glorot(rng, shape[0], shape[1], shape)   # orthogonal; glorot here)
        elif name.endswith("/bias"):
            W[name] = (rng.uniform(-0.1, 0.1, size=shape).astype(np.float32) if for_test
                       else np.zeros(shape, np.float32))
        elif name.endswith("/alpha"):
            W[name] = (rng.uniform(0.0, 0.5, size=shape).astype(np.float32) if for_test
                       else np.zeros(shape, np.float32))
        else:
            raise AssertionError(name)
    if for_test:
        for kname, rows in numeric_rows(spec).items():
            if kname in W:
                W[kname][rows, :] /= _NUMERIC_SCALE[:, None]
        # one-hot first-order weights: glorot over a 30k-wide fan-in is ~0.01; widen so
        # the scalar gathers are visible in the logit
        onehot_rows = {"deepfm": ("dense_2/kernel", slice(0, spec.fm1_width)),
                       "widendeep": ("dense_2/kernel", slice(spec.hidden[-1] if spec.hidden else 0, None)),
                       "deepfm_v2": ("first_cat/kernel", slice(None))}.get(spec.model)
        if onehot_rows is not None and onehot_rows[0] in W:
            k = W[onehot_rows[0]]
            n = k[onehot_rows[1]].shape
            k[onehot_rows[1]] = rng.uniform(-0.5, 0.5, size=n).astype(np.float32)
    return W


def aux_weight_shapes(spec: ModelSpec) -> List[Tuple[str, Tuple[int, ...]]]:
    """DIEN's optional auxiliary-head group (`auxiliary_loss_layer`, DIEN.py:261-270): two Dense(32, sigmoid)
    over [g_t | e] and two Dense(1, sigmoid), for the positive and the negative next item.  A DIEN model takes
    all eight or none; without them it serves `y_pred` only.  Kept apart from `weight_shapes` so that the
    model's base inventory - and the seeded draws of `init_weights` - stay what they are."""
    if spec.model != "dien":
        raise ValueError("the auxiliary-head weights belong to DIEN, not %r" % spec.model)
    E = spec.emb_dim
    out: List[Tuple[str, Tuple[int, ...]]] = []
    for side in ("pos", "neg"):                 # DIEN.py:265-268
        out += [("aux_%s_dense/kernel" % side, (2 * E, 32)), ("aux_%s_dense/bias" % side, (32,)),
                ("aux_%s_out/kernel" % side, (32, 1)), ("aux_%s_out/bias" % side, (1,))]
    return out


def init_aux_weights(spec: ModelSpec, seed: int = 0) -> Dict[str, np.ndarray]:
    """Seeded auxiliary-head weights with Keras's Dense defaults: glorot_uniform kernels, zero biases.  The draws
    come from their own generator, so adding the group leaves `init_weights(spec, seed)` unchanged."""
    rng = np.random.default_rng(seed)
    return {name: (_glorot(rng, shape[0], shape[1], shape) if name.endswith("/kernel")
                   else np.zeros(shape, np.float32))
            for name, shape in aux_weight_shapes(spec)}


def check_weights(spec: ModelSpec, W: Dict[str, np.ndarray], skip: Tuple[str, ...] = ()) -> None:
    for name, shape in weight_shapes(spec):
        if name in skip:
            continue
        if name not in W:
            raise KeyError("missing weight tensor %r for model %s" % (name, spec.model))
        if tuple(W[name].shape) != shape:
            raise ValueError("weight %r has shape %s, expected %s"
                             % (name, tuple(W[name].shape), shape))
        if W[name].dtype != np.float32:
            raise ValueError("weight %r must be float32" % name)


def has_aux_weights(spec: ModelSpec, W) -> bool:
    """True when `W` carries DIEN's auxiliary-head group (checked: all eight tensors with their shapes, float32),
    False when it carries none of it; KeyError / ValueError for a partial or malformed group."""
    if spec.model != "dien":
        return False
    shapes = aux_weight_shapes(spec)
    present = [n for n, _ in shapes if n in W]
    if not present:
        return False
    for name, shape in shapes:
        if name not in W:
            raise KeyError("missing weight tensor %r: the auxiliary-head group is all eight tensors or none" % name)
        a = W[name]
        if tuple(a.shape) != shape:
            raise ValueError("weight %r has shape %s, expected %s" % (name, tuple(a.shape), shape))
        if not isinstance(a, np.ndarray) or a.dtype != np.float32:
            raise ValueError("weight %r must be a float32 host array" % name)
    return True
