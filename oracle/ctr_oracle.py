"""CPU oracle: numpy restatement of the SparrowRecSys Keras CTR graphs.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT.  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s CPU-baseline / `--impl reference` legs
may import it; the product path (`sparrowrecsys_b200`, `tfrecmodel`) never does
and fails loudly when the CUDA library is missing.

PARITY UNPINNED: the reference's arithmetic lives in TensorFlow (README.md:11
"TensorFlow 2.0+", exports written by TF 2.0.0 / keras 2.2.4-tf), which is not
vendored under /root/reference, is not installed in this image and cannot be
installed (no network); the reference ships no tests.  This file restates the
graphs from the reference scripts plus the TF semantics recorded in SURVEY.md
section 8a.  What *does* anchor it: the reference's shipped trained weights
(`modeldata/neuralcf/{001,002}`, `modeldata/MLPRec/005`) on the bundled
`testSamples.csv` rows reproduce the known answers recorded in SURVEY.md
section 8c (tests/test_oracle_golden.py), computed by an independent restatement,
and - round 2 - the outputs of the reference's own serialised `serving_default`
functions (`saved_model.pb` of those three exports, evaluated node by node by
`oracle/savedmodel_graph.py`; `tests/golden/savedmodel_graph_vectors.json`): for
`neuralcf_forward` and the shipped form of `twotowers_forward` the graph wiring is
TensorFlow's, not a reading of the script.  The other graphs stay unpinned.

All paths below are relative to
/root/reference/TFRecModel/src/com/sparrowrecsys/offline/tensorflow/.

Conventions: `spec` is any object with the attributes of
`sparrowrecsys_b200.spec.ModelSpec`; `W` maps the canonical tensor names of
`sparrowrecsys_b200.weights.weight_shapes` to float32 arrays in the reference's
(Keras) shapes; `feats` is the dict that `model.predict` receives (1-D columns;
genres as str/bytes).  Every forward returns `(prob[B,1], logit[B,1])`;
`dtype=np.float64` runs the same graph in double to bound reassociation error.
"""
from __future__ import annotations

import numpy as np

GENRE_VOCAB = ("Film-Noir", "Action", "Adventure", "Horror", "Romance", "War", "Comedy",
               "Western", "Documentary", "Sci-Fi", "Drama", "Thriller", "Crime", "Fantasy",
               "Animation", "IMAX", "Mystery", "Children", "Musical")   # DIN.py:70-72
_GIDX = {g: i for i, g in enumerate(GENRE_VOCAB)}


# ----------------------------------------------------------------------------------
# feature-column primitives (SURVEY.md section 8a items 1-8)
# ----------------------------------------------------------------------------------
def _col(feats, key):
    a = np.asarray(feats[key])
    return a[:, 0] if a.ndim == 2 else a


def numeric(feats, key, dtype):
    """tf.feature_column.numeric_column: cast to float32 -> [B,1]."""
    return _col(feats, key).astype(np.float32).astype(dtype)[:, None]


def genre_index(feats, key):
    """categorical_column_with_vocabulary_list: position in vocab, OOV/"" -> -1."""
    a = _col(feats, key)
    if a.dtype.kind in "iu":
        return a.astype(np.int64)
    out = np.empty(a.shape[0], np.int64)
    for i, v in enumerate(a):
        if isinstance(v, bytes):
            v = v.decode()
        out[i] = _GIDX.get(v, -1)
    return out


def identity_ids(feats, key, num_buckets):
    """categorical_column_with_identity: asserts 0 <= id < num_buckets."""
    a = _col(feats, key).astype(np.int64)
    if a.size and (a.min() < 0 or a.max() >= num_buckets):
        raise ValueError("%s out of range [0,%d)" % (key, num_buckets))
    return a


def embedding_column(table, ids, dtype):
    """embedding_column(combiner='mean') on one id per row: the row; id -1
    (missing / OOV after pruning) -> all-zero vector."""
    t = table.astype(dtype)
    out = t[np.maximum(ids, 0)]
    out[ids < 0] = 0
    return out


def indicator_weight(kernel_rows, ids, dtype):
    """indicator_column one-hot times a [width,1] kernel slice == scalar gather;
    empty (id -1) -> 0."""
    w = kernel_rows.astype(dtype)[np.maximum(ids, 0), 0]
    w[ids < 0] = 0
    return w[:, None]


def dense(x, W, prefix, act=None):
    """tf.keras.layers.Dense: x @ kernel + bias, contracting the last axis."""
    y = x @ W[prefix + "/kernel"].astype(x.dtype) + W[prefix + "/bias"].astype(x.dtype)
    if act == "relu":
        y = np.maximum(y, 0)
    elif act == "sigmoid":
        y = sigmoid(y)
    return y


def prelu(x, alpha):
    """tf.keras.layers.PReLU: relu(x) - alpha * relu(-x); alpha has the input's
    shape without the batch axis."""
    a = alpha.astype(x.dtype)
    return np.maximum(x, 0) - a * np.maximum(-x, 0)


def sigmoid(x):
    out = np.empty_like(x)
    pos = x >= 0
    out[pos] = 1.0 / (1.0 + np.exp(-x[pos]))
    ex = np.exp(x[~pos])
    out[~pos] = ex / (1.0 + ex)
    return out


# ----------------------------------------------------------------------------------
# W&D crossed column hash (WideNDeep.py:72-73)
# ----------------------------------------------------------------------------------
_M64 = (1 << 64) - 1
_K_MUL = 0xC6A4A7935BD1E995


def _shift_mix(v):
    return v ^ (v >> 47)


def fingerprint_cat64(fp1, fp2):
    """tensorflow/core/platform/fingerprint.h FingerprintCat64 (restated; TF source
    not vendored -- SURVEY.md section 8c residual risk)."""
    result = fp1 ^ _K_MUL
    result ^= (_shift_mix((fp2 * _K_MUL) & _M64) * _K_MUL) & _M64
    result = (result * _K_MUL) & _M64
    result = (_shift_mix(result) * _K_MUL) & _M64
    result = _shift_mix(result)
    return result & _M64


def crossed_bucket(movie_id, rated_movie, num_buckets=10000, hash_key=0xDECAFCAFFE):
    """crossed_column([movieId, userRatedMovie1], 10000): SparseCross with
    hashed_output, leaf order movieId then userRatedMovie1."""
    h = fingerprint_cat64(hash_key, int(movie_id) & _M64)
    h = fingerprint_cat64(h, int(rated_movie) & _M64)
    return h % num_buckets


def crossed_bucket_array(movie_ids, rated, num_buckets=10000):
    return np.array([crossed_bucket(int(a), int(b), num_buckets)
                     for a, b in zip(movie_ids, rated)], dtype=np.int64)


# ----------------------------------------------------------------------------------
# graphs
# ----------------------------------------------------------------------------------
def _embmlp_input(spec, W, feats, dtype):
    """DenseFeatures(numerical_columns + categorical_columns), EmbeddingMLP.py:73 /
    WideNDeep.py:101 -- concat sorted by column name."""
    mid = identity_ids(feats, "movieId", spec.n_movies)
    uid = identity_ids(feats, "userId", spec.n_users)
    parts = [numeric(feats, "movieAvgRating", dtype)]
    for k in (1, 2, 3):
        parts.append(embedding_column(W["movieGenre%d_embedding" % k],
                                      genre_index(feats, "movieGenre%d" % k), dtype))
    parts.append(embedding_column(W["movieId_embedding"], mid, dtype))
    parts += [numeric(feats, k, dtype) for k in
              ("movieRatingCount", "movieRatingStddev", "releaseYear", "userAvgRating")]
    for k in (1, 2, 3, 4, 5):
        parts.append(embedding_column(W["userGenre%d_embedding" % k],
                                      genre_index(feats, "userGenre%d" % k), dtype))
    parts.append(embedding_column(W["userId_embedding"], uid, dtype))
    parts += [numeric(feats, k, dtype) for k in ("userRatingCount", "userRatingStddev")]
    return np.concatenate(parts, axis=1)


def embeddingmlp_forward(spec, W, feats, dtype=np.float32):
    """EmbeddingMLP.py:72-77."""
    x = _embmlp_input(spec, W, feats, dtype)
    x = dense(x, W, "dense", "relu")
    x = dense(x, W, "dense_1", "relu")
    z = dense(x, W, "dense_2")
    return sigmoid(z), z


def widendeep_forward(spec, W, feats, dtype=np.float32):
    """WideNDeep.py:101-107: [deep(128) | one-hot_10000(cross)] -> Dense(1,sigmoid)."""
    x = _embmlp_input(spec, W, feats, dtype)
    x = dense(x, W, "dense", "relu")
    deep = dense(x, W, "dense_1", "relu")
    mid = identity_ids(feats, "movieId", spec.n_movies)
    rated = identity_ids(feats, "userRatedMovie1", spec.n_movies)
    bucket = crossed_bucket_array(mid, rated, spec.cross_buckets)
    K = W["dense_2/kernel"].astype(dtype)
    h1 = deep.shape[1]
    z = deep @ K[:h1] + K[h1 + bucket] + W["dense_2/bias"].astype(dtype)
    return sigmoid(z), z


def neuralcf_forward(spec, W, feats, dtype=np.float32):
    """neural_cf_model_1, NeuralCF.py:45-53: concat(item, user) -> Dense relu.. -> Dense(1,sigmoid)."""
    item = embedding_column(W["movieId_embedding"], identity_ids(feats, "movieId", spec.n_movies), dtype)
    user = embedding_column(W["userId_embedding"], identity_ids(feats, "userId", spec.n_users), dtype)
    x = np.concatenate([item, user], axis=1)
    n = len(spec.hidden)
    for i in range(n):
        x = dense(x, W, "dense_%d" % i, "relu")
    z = dense(x, W, "dense_%d" % n)
    return sigmoid(z), z


def twotowers_forward(spec, W, feats, dtype=np.float32):
    """neural_cf_model_2, NeuralCF.py:57-70.  With `final_dense=False` (the shipped
    MLPRec/005 export) the output is the raw Dot(axes=1) and `prob == logit`."""
    item = embedding_column(W["movieId_embedding"], identity_ids(feats, "movieId", spec.n_movies), dtype)
    user = embedding_column(W["userId_embedding"], identity_ids(feats, "userId", spec.n_users), dtype)
    for i in range(len(spec.hidden)):
        item = dense(item, W, "item_dense_%d" % i, "relu")
        user = dense(user, W, "user_dense_%d" % i, "relu")
    d = np.sum(item * user, axis=1, keepdims=True)
    if not spec.final_dense:
        return d, d
    z = dense(d, W, "dense_out")
    return sigmoid(z), z


def deepfm_forward(spec, W, feats, dtype=np.float32):
    """DeepFM.py:91-113."""
    mid = identity_ids(feats, "movieId", spec.n_movies)
    uid = identity_ids(feats, "userId", spec.n_users)
    ig_i = genre_index(feats, "movieGenre1")
    ug_i = genre_index(feats, "userGenre1")
    item = embedding_column(W["fm_movieId_embedding"], mid, dtype)          # :91
    user = embedding_column(W["fm_userId_embedding"], uid, dtype)           # :92
    ig = embedding_column(W["fm_movieGenre1_embedding"], ig_i, dtype)       # :93
    ug = embedding_column(W["fm_userGenre1_embedding"], ug_i, dtype)        # :94
    dot = lambda a, b: np.sum(a * b, axis=1, keepdims=True)
    dots = [dot(item, user), dot(ig, ug), dot(ig, user), dot(item, ug)]     # :100-103
    # deep DenseFeatures (own tables), sorted concat                        # :106
    deep = np.concatenate([
        numeric(feats, "movieAvgRating", dtype),
        embedding_column(W["deep_movieId_embedding"], mid, dtype),
        numeric(feats, "movieRatingCount", dtype),
        numeric(feats, "movieRatingStddev", dtype),
        numeric(feats, "releaseYear", dtype),
        numeric(feats, "userAvgRating", dtype),
        embedding_column(W["deep_userId_embedding"], uid, dtype),
        numeric(feats, "userRatingCount", dtype),
        numeric(feats, "userRatingStddev", dtype)], axis=1)
    deep = dense(deep, W, "dense", "relu")
    deep = dense(deep, W, "dense_1", "relu")
    # final Dense over [fm1 one-hots (sorted: movieGenre1|movieId|userGenre1|userId) | 4 dots | deep]
    K = W["dense_2/kernel"]
    G, Vm = spec.n_genres, spec.n_movies
    o_mg, o_m, o_ug, o_u = 0, G, G + Vm, G + Vm + G
    o_d = spec.fm1_width
    z = (indicator_weight(K[o_mg:o_m], ig_i, dtype) + indicator_weight(K[o_m:o_ug], mid, dtype)
         + indicator_weight(K[o_ug:o_u], ug_i, dtype) + indicator_weight(K[o_u:o_d], uid, dtype))
    Kd = K.astype(dtype)
    z = z + np.concatenate(dots, axis=1) @ Kd[o_d:o_d + 4] + deep @ Kd[o_d + 4:] \
        + W["dense_2/bias"].astype(dtype)
    return sigmoid(z), z


def deepfm_v2_forward(spec, W, feats, dtype=np.float32):
    """DeepFM_v2.py:98-155."""
    mid = identity_ids(feats, "movieId", spec.n_movies)
    uid = identity_ids(feats, "userId", spec.n_users)
    ig_i = genre_index(feats, "movieGenre1")
    ug_i = genre_index(feats, "userGenre1")
    G, Vm = spec.n_genres, spec.n_movies
    K1 = W["first_cat/kernel"]
    first_cat = (indicator_weight(K1[0:G], ig_i, dtype)
                 + indicator_weight(K1[G:G + Vm], mid, dtype)
                 + indicator_weight(K1[G + Vm:2 * G + Vm], ug_i, dtype)
                 + indicator_weight(K1[2 * G + Vm:], uid, dtype)
                 + W["first_cat/bias"].astype(dtype))                        # :98-99
    nums = np.concatenate([numeric(feats, k, dtype) for k in (
        "movieAvgRating", "movieRatingCount", "movieRatingStddev", "releaseYear",
        "userAvgRating", "userRatingCount", "userRatingStddev")], axis=1)    # sorted deep_columns
    first_num = dense(nums, W, "first_num")                                  # :100-101
    first = first_cat + first_num                                            # :104
    fields = [                                                               # :106-116
        dense(embedding_column(W["movieGenre1_embedding"], ig_i, dtype), W, "proj_movieGenre1"),
        dense(embedding_column(W["movieId_embedding"], mid, dtype), W, "proj_movieId"),
        dense(embedding_column(W["userGenre1_embedding"], ug_i, dtype), W, "proj_userGenre1"),
        dense(embedding_column(W["userId_embedding"], uid, dtype), W, "proj_userId"),
        dense(nums, W, "proj_num"),                                          # :118-120
    ]
    F = np.stack(fields, axis=1)                                             # [B,5,P] :121
    deep = F.reshape(F.shape[0], -1)                                         # Flatten :124
    deep = dense(deep, W, "deep", "relu")
    deep = dense(deep, W, "deep_1", "relu")
    s = F.sum(axis=1)
    fm = s * s - (F * F).sum(axis=1)                                         # :147-152 (no 1/2)
    z = dense(np.concatenate([first, fm, deep], axis=1), W, "out")           # :154-155
    return sigmoid(z), z


def din_history_keys(T):
    return sorted("userRatedMovie%d" % k for k in range(1, T + 1))


def din_forward(spec, W, feats, dtype=np.float32, defect=None, chunk=32):
    """DIN.py:125-167.  Sigmoid-gated *sum* pooling (no softmax), history id 0 is
    an ordinary table row (mask_zero has no numerical effect), ids pass through a
    float32 numeric_column before the Embedding layer casts them back to int32.

    `defect` (mutants for the tests; a kernel stages `chunk` positions at a time):
    "last" leaves position T - 1 out of the pool, "chunk" a partial last chunk,
    "pad" every padding position (id 0), and "alpha" reads position t's PReLU alpha
    at t mod chunk."""
    E, T = spec.emb_dim, spec.hist_len
    cand_f = numeric(feats, "movieId", np.float32)                           # :95,125
    hist_f = np.concatenate([numeric(feats, k, np.float32) for k in din_history_keys(T)],
                            axis=1)                                          # :97-103,126
    cand = cand_f.astype(np.int32)[:, 0]
    hist = hist_f.astype(np.int32)
    if cand.min() < 0 or max(cand.max(), hist.max()) >= spec.n_movies or hist.min() < 0:
        raise ValueError("movie id out of range")
    tab = W["embedding"].astype(dtype)
    H = tab[hist]                                                            # [B,T,E] :134
    C = tab[cand]                                                            # [B,E]   :136-137
    Cr = np.repeat(C[:, None, :], T, axis=1)                                 # :139
    A = np.concatenate([H - Cr, H, Cr, H * Cr], axis=-1)                     # :141-147
    a = dense(A, W, "au_dense")                                              # :149
    alpha = W["au_prelu/alpha"]
    if defect == "alpha":
        alpha = alpha[np.arange(T) % chunk]
    a = prelu(a, alpha)                                                      # :150 alpha [T,32]
    w = dense(a, W, "au_out", "sigmoid")[..., 0]                             # :151-152 [B,T]
    if defect == "last":
        w[:, T - 1] = 0
    elif defect == "chunk":
        w[:, T - T % chunk:] = 0
    elif defect == "pad":
        w[hist == 0] = 0
    pooled = (H * w[:, :, None]).sum(axis=1)                                 # :153-158
    uid = identity_ids(feats, "userId", spec.n_users)
    user_profile = np.concatenate([                                          # :108-114,127 sorted
        numeric(feats, "userAvgRating", dtype),
        embedding_column(W["userGenre1_embedding"], genre_index(feats, "userGenre1"), dtype),
        embedding_column(W["userId_embedding"], uid, dtype),
        numeric(feats, "userRatingCount", dtype),
        numeric(feats, "userRatingStddev", dtype)], axis=1)
    context = np.concatenate([                                               # :117-123,128 sorted
        numeric(feats, "movieAvgRating", dtype),
        embedding_column(W["movieGenre1_embedding"], genre_index(feats, "movieGenre1"), dtype),
        numeric(feats, "movieRatingCount", dtype),
        numeric(feats, "movieRatingStddev", dtype),
        numeric(feats, "releaseYear", dtype)], axis=1)
    x = np.concatenate([user_profile, pooled, C, context], axis=1)           # :161-162
    x = prelu(dense(x, W, "dense"), W["prelu/alpha"])                        # :163-164
    x = prelu(dense(x, W, "dense_1"), W["prelu_1/alpha"])                    # :165-166
    z = dense(x, W, "dense_2")                                               # :167
    return sigmoid(z), z


def dien_forward(spec, W, feats, dtype=np.float32, defect=None):
    """DIEN.py:154-256, the `y_pred` output (the auxiliary-loss head, :259-292, only feeds
    `add_loss` and is not part of the prediction).

    Two things differ from DIN's use of the same `Embedding(mask_zero=True)` layer:
    * the mask IS consumed here: `GRU(...)(user_behaviors_emb_layer)` (:169) receives the
      Embedding's mask (`inputs != 0`), and Keras' masked RNN step carries state and output
      over a masked position (`K.rnn`: `where(mask, new, old)`, previous output = zeros before
      the first valid step) - so a padded slot repeats the last hidden state;
    * the AUGRU's initial state is `GlorotUniform()(shape=(1, E))` evaluated inside `call`
      (:235-236), i.e. a fresh random vector per forward pass: the reference's predictions
      are not reproducible.  Here that vector is the stored tensor `augru_h0` [1,E].

    GRU: Keras defaults - gate order z | r | h, sigmoid / tanh, `reset_after=True`:
      mx = x.K + b[0];  mh = h.U + b[1];  z = s(mx_z + mh_z);  r = s(mx_r + mh_r)
      hh = tanh(mx_h + r * mh_h);  h' = z * h + (1 - z) * hh
    Attention (:172-195): s_t = sigmoid(Dense1(sigmoid(Dense32(g_t * c)))) per position.
    AUGRU (:204-245), per step with x = g_t, state u:
      r = s(Act_r(In_r(x) + Hid_r(u)));  z = s(Act_z(In_z(x) + Hid_z(u)))
      hn = tanh(Act_h(In_h(x) + Hid_h(u * z)));  a = s_t * r;  u' = (1 - a) * u + a * hn
    (`In` Dense with bias, `Hid` Dense without, `Act` Dense with bias and the activation).
    Top (:250-256): [u_T | candidate | user_profile | context] -> 128 PReLU -> 64 PReLU -> 1.

    `defect` (mutants for the tests): "last" stops both recurrences before position T - 1,
    "mask" runs the GRU over padding (id 0) as over any row."""
    E, T = spec.emb_dim, spec.hist_len
    cand_f = numeric(feats, "movieId", np.float32)                           # :96,154
    hist_f = np.concatenate([numeric(feats, k, np.float32) for k in din_history_keys(T)],
                            axis=1)                                          # :99-105,155
    cand = cand_f.astype(np.int32)[:, 0]
    hist = hist_f.astype(np.int32)
    if cand.min() < 0 or max(cand.max(), hist.max()) >= spec.n_movies or hist.min() < 0:
        raise ValueError("movie id out of range")
    mask = hist_f != 0                                                       # Embedding.compute_mask
    if defect == "mask":
        mask[:] = True
    steps = T - 1 if defect == "last" else T
    tab = W["embedding"].astype(dtype)
    X = tab[hist]                                                            # [B,T,E] :163
    C = tab[cand]                                                            # [B,E]   :164,167
    B = cand.shape[0]
    K, U = W["gru/kernel"].astype(dtype), W["gru_recurrent/kernel"].astype(dtype)
    bx, bh = W["gru/bias"].astype(dtype)
    h = np.zeros((B, E), dtype)
    G = np.zeros((B, T, E), dtype)
    for t in range(steps):                                                   # :169
        mx = X[:, t] @ K + bx
        mh = h @ U + bh
        z = sigmoid(mx[:, :E] + mh[:, :E])
        r = sigmoid(mx[:, E:2 * E] + mh[:, E:2 * E])
        hh = np.tanh(mx[:, 2 * E:] + r * mh[:, 2 * E:])
        hn = z * h + (1 - z) * hh
        h = np.where(mask[:, t, None], hn, h)
        G[:, t] = h
    att = dense(dense(G * C[:, None, :], W, "att_dense", "sigmoid"), W, "att_out", "sigmoid")[..., 0]

    def gate(g, x, hid):                                                     # :204-219
        pre = dense(x, W, "augru_%s_input" % g) + hid @ W["augru_%s_hidden/kernel" % g].astype(dtype)
        return dense(pre, W, "augru_%s_act" % g)
    u = np.repeat(W["augru_h0"].astype(dtype), B, axis=0)                    # :235-236 (stored)
    for t in range(steps):                                                   # :237-243
        x = G[:, t]
        r = sigmoid(gate("r", x, u))
        z = sigmoid(gate("z", x, u))
        hn = np.tanh(gate("h", x, u * z))
        a = att[:, t, None] * r
        u = (1 - a) * u + a * hn
    uid = identity_ids(feats, "userId", spec.n_users)
    user_profile = np.concatenate([                                          # :124-130,157 sorted
        numeric(feats, "userAvgRating", dtype),
        embedding_column(W["userGenre1_embedding"], genre_index(feats, "userGenre1"), dtype),
        embedding_column(W["userId_embedding"], uid, dtype),
        numeric(feats, "userRatingCount", dtype),
        numeric(feats, "userRatingStddev", dtype)], axis=1)
    context = np.concatenate([                                               # :133-139,158 sorted
        numeric(feats, "movieAvgRating", dtype),
        embedding_column(W["movieGenre1_embedding"], genre_index(feats, "movieGenre1"), dtype),
        numeric(feats, "movieRatingCount", dtype),
        numeric(feats, "movieRatingStddev", dtype),
        numeric(feats, "releaseYear", dtype)], axis=1)
    x = np.concatenate([u, C, user_profile, context], axis=1)                # :250
    x = prelu(dense(x, W, "dense"), W["prelu/alpha"])                        # :252-253
    x = prelu(dense(x, W, "dense_1"), W["prelu_1/alpha"])                    # :254-255
    zlogit = dense(x, W, "dense_2")                                          # :256
    return sigmoid(zlogit), zlogit


FORWARD = {
    "embeddingmlp": embeddingmlp_forward,
    "widendeep": widendeep_forward,
    "neuralcf": neuralcf_forward,
    "twotowers": twotowers_forward,
    "deepfm": deepfm_forward,
    "deepfm_v2": deepfm_v2_forward,
    "din": din_forward,
    "dien": dien_forward,
}


def forward(spec, W, feats, dtype=np.float32):
    return FORWARD[spec.model](spec, W, feats, dtype)


def predict(spec, W, feats, batch_size=None, dtype=np.float32):
    """`model.predict(x)` (e.g. DIN.py:185): float32 [N,1]; optionally in batches
    like the Keras predict loop (which uses the dataset's batch size, 12)."""
    n = len(_col(feats, "movieId"))
    if batch_size is None or batch_size >= n:
        return forward(spec, W, feats, dtype)[0].astype(np.float32)
    outs = []
    for lo in range(0, n, batch_size):
        sub = {k: np.asarray(v)[lo:lo + batch_size] for k, v in feats.items()}
        outs.append(forward(spec, W, sub, dtype)[0])
    return np.concatenate(outs, axis=0).astype(np.float32)


# ----------------------------------------------------------------------------------
# helpers around the path (not reference graphs)
# ----------------------------------------------------------------------------------
def fill_uniform(indices, seed, lo, hi):
    """numpy replica of srs_fill_uniform (csrc/util.cu): element i of the synthetic
    device-initialised table; `indices` is an int array of flat element indices."""
    i = np.asarray(indices, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (i + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    u = (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    span = np.float32(np.float32(hi) - np.float32(lo))
    return (np.float32(lo) + span * u).astype(np.float32)


def cosine_similarity(query, cands):
    """online/model/Embedding.java:33-47: float products accumulated in double."""
    q = np.asarray(query, np.float32)
    c = np.asarray(cands, np.float32)
    dot = (q[None, :] * c).astype(np.float64).sum(axis=1)
    n1 = (q * q).astype(np.float64).sum()
    n2 = (c * c).astype(np.float64).sum(axis=1)
    return dot / (np.sqrt(n1) * np.sqrt(n2))


def java_double_compare(a, b):
    """java.lang.Double.compare, the order `Map.Entry.comparingByValue` sorts boxed Doubles
    by: numeric order, then -0.0 < 0.0, and NaN (canonicalised) above +infinity."""
    import struct
    a, b = float(a), float(b)
    if a < b:
        return -1
    if a > b:
        return 1
    bits = lambda x: 0x7FF8000000000000 if x != x else struct.unpack("<q", struct.pack("<d", x))[0]
    ba, bb = bits(a), bits(b)
    return 0 if ba == bb else (-1 if ba < bb else 1)


def rank_topk(scores, k):
    """The ranker tail of online/recprocess/RecForYouProcess.java:92-94 (same in
    SimilarMovieProcess.java:133-135) and the `subList(0, size)` of getRecList (:56-59):
    candidates sorted by score with `comparingByValue(Comparator.reverseOrder())`, first
    `size` kept.  The Java stream sort is stable over the HashMap's (unspecified) iteration
    order; here equal scores keep candidate order.  Returns (positions int32, scores float32).
    Pure-Python comparison sort: meant for the few thousand candidates a request ranks."""
    from functools import cmp_to_key
    s = np.asarray(scores, np.float32).reshape(-1)
    d = [float(v) for v in s]
    order = sorted(range(len(d)), key=cmp_to_key(lambda i, j: java_double_compare(d[j], d[i])))
    order = np.asarray(order[:max(int(k), 0)], np.int32)
    return order, s[order]
