"""Float64 emulation of the bf16 split arithmetic of the tensor-core kernels.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT (see oracle/ctr_oracle.py).

The tensor-core kernels split every MMA operand x (an fp32 value) into `hi = bf16(x)` and
`lo = bf16(x - hi)`, both rounded to nearest-even as `__float2bfloat16_rn` does, and accumulate the
products in fp32.  Which products each stage forms, read off the kernels:

* `din_wg.cu` activation unit: per batch row r, `W_r = (Wsub + Wh) + diag(c_r) Wp` is formed in fp32
  (one fmaf per element) and split; the history rows H come split from the pre-split table.  Three
  products: `H_hi W_hi + H_lo W_hi + H_hi W_lo` (stage "au").
* `din_wg.cu` pooling: `sum_t w_t h_t` with `h = hi + lo` read back from the same tile (stage "pool").
* The MLP stages - `din_wg.cu`'s top MLP at EP = 32, `embmlp_tc.cu` and `deepfm_tc.cu`: both W images
  (hi and lo) against the stacked `[X_hi | X_lo]` operand, so all four products (stages "mlp1" and
  "mlp2", the two Dense layers).  The 7 raw-scale numerics never enter an MMA: their contribution is
  added in fp32 in the layer-1 epilogue.

Everything else - gathers, the activation-unit constant, PReLU, the gate, the last Dense(1), the FM
and wide parts, and din_wg's CUDA-core top MLP at EP = 64 - is evaluated in float64 here, so the
only error the emulation carries is the split's.

`forward(spec, W, feats, defect=None)` returns float64 `(prob[B,1], logit[B,1])` like
`ctr_oracle.forward`.  A `Defect` removes one thing from one stage, optionally confined to one path
of the kernel (rows after the first tile, late or last history positions, a K range), so that a
test can ask whether its tolerance would see a kernel that lost or misplaced a lo half there.
"""
from __future__ import annotations

import dataclasses
from typing import Optional, Tuple

import numpy as np

from . import ctr_oracle as O

NUMERIC_KEYS = ("movieAvgRating", "movieRatingCount", "movieRatingStddev", "releaseYear",
                "userAvgRating", "userRatingCount", "userRatingStddev")

AU_TERMS = ("hh", "lh", "hl")              # din_wg activation unit: X = H (history), W = W_r
MLP_TERMS = ("hh", "lh", "hl", "ll")       # both W images against [X_hi | X_lo]
DROPS = {"x_lo": ("lh", "ll"), "w_lo": ("hl", "ll"), "lo": ("lh", "hl", "ll")}


def bf16(x) -> np.ndarray:
    """`__float2bfloat16_rn` of float32 values (round to nearest, ties to even), as float64."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32).astype(np.float64)


def split(x) -> Tuple[np.ndarray, np.ndarray]:
    """(hi, lo) of the fp32 value of x: `hi = bf16(x)`, `lo = bf16(x - hi)` (the difference is exact in fp32)."""
    x32 = np.asarray(x, np.float32)
    hi = bf16(x32)
    lo = bf16((x32.astype(np.float64) - hi).astype(np.float32))
    return hi, lo


@dataclasses.dataclass(frozen=True)
class Defect:
    """One thing removed from one stage.

    stage:  "au" | "pool" | "mlp1" | "mlp2".
    drop:   "x_lo" (the activation / history operand's lo plane), "w_lo" (the weight operand's lo
            plane), "lo" (both: hi.hi only), or - mlp1 only - "numerics" (the 7 numerics rounded to
            bf16 hi instead of kept fp32).  The pool stage has only "lo" (h = hi).
    rows_from: the defect hits batch rows >= rows_from only (rows after the first tile / super-group).
    t_from:    au / pool: history positions >= t_from only (64: the ring of tiles after the first;
               64 * (n_tiles - 1): the last partial tile).
    k:         (k0, k1): operand K columns k0 <= k < k1 only - au: embedding elements of each plane;
               mlp1: columns of the kernel's X tile; mlp2: hidden units."""
    stage: str
    drop: str
    rows_from: int = 0
    t_from: int = 0
    k: Optional[Tuple[int, int]] = None

    def __post_init__(self):
        assert self.stage in ("au", "pool", "mlp1", "mlp2"), self.stage
        ok = {"au": DROPS, "pool": ("lo",), "mlp1": (*DROPS, "numerics"), "mlp2": DROPS}[self.stage]
        assert self.drop in ok, (self.stage, self.drop)


def _hit(defect, stage, shape, row0, pos_axis=None, k_axis=-1):
    """Bool mask over an operand of `shape` (axis 0 = batch rows starting at row0): True where `defect`
    removes something at this stage; None when it does not touch the stage."""
    if defect is None or defect.stage != stage:
        return None
    m = np.ones(shape, bool)
    rows = row0 + np.arange(shape[0])
    m &= (rows >= defect.rows_from).reshape((-1,) + (1,) * (len(shape) - 1))
    if pos_axis is not None and defect.t_from:
        view = [1] * len(shape)
        view[pos_axis] = shape[pos_axis]
        m &= (np.arange(shape[pos_axis]) >= defect.t_from).reshape(view)
    if defect.k is not None:
        view = [1] * len(shape)
        view[k_axis] = shape[k_axis]
        k = np.arange(shape[k_axis])
        m &= ((k >= defect.k[0]) & (k < defect.k[1])).reshape(view)
    return m


def split_product(x, w, terms, subscripts, hit=None, drop=None):
    """sum over `terms` ("hh": x_hi w_hi, "lh": x_lo w_hi, ...) of einsum(subscripts, x_a, w_b), with
    x_a zeroed where `hit` in the terms `drop` removes."""
    xs, ws = dict(zip("hl", split(x))), dict(zip("hl", split(w)))
    out = 0.0
    for t in terms:
        xa = xs[t[0]]
        if hit is not None and t in DROPS.get(drop, ()):
            xa = np.where(hit, 0.0, xa)
        out = out + np.einsum(subscripts, xa, ws[t[1]], optimize=True)
    return out


def _mlp_layer(x, w, stage, defect, row0):
    hit = _hit(defect, stage, x.shape, row0)
    return split_product(x, w, MLP_TERMS, "rk,ku->ru", hit, defect.drop if hit is not None else None)


def _numerics(feats):
    return np.concatenate([O.numeric(feats, k, np.float64) for k in NUMERIC_KEYS], axis=1)


def _numeric_term(feats, w_num, defect, row0):
    """The layer-1 epilogue's fp32 numerics term; rounded to bf16 under the "numerics" defect."""
    nums = _numerics(feats)
    hit = _hit(defect, "mlp1", nums.shape[:1] + (1,), row0)
    if hit is not None and defect.drop == "numerics":
        nums = np.where(hit, bf16(nums), nums)
    return nums @ w_num.astype(np.float64)


def _pad_rows(a, n):
    out = np.zeros((n,) + a.shape[1:], a.dtype)
    out[:a.shape[0]] = a
    return out


# ---- din_wg_kernel<EP> -------------------------------------------------------------------------------
def din_tile_columns(E, EP):
    """Row of `dense/kernel` feeding each column of din_wg's top-MLP X tile
    [userGenre1 | userId | pooled | candidate | movieGenre1] (EP columns each, -1 = zero padding), and
    the rows of the 7 numerics in NUMERIC_KEYS order (csrc/placement.h place_din)."""
    base = 3 + 4 * E
    starts = (1, 1 + E, 3 + 2 * E, 3 + 3 * E, base + 1)
    cols = np.full(5 * EP, -1, np.int64)
    for b, s in enumerate(starts):
        cols[b * EP:b * EP + E] = s + np.arange(E)
    nums = np.array([base, base + 1 + E, base + 2 + E, base + 3 + E, 0, 1 + 2 * E, 2 + 2 * E])
    return cols, nums


def _rows_of(k, cols):
    out = np.zeros((cols.shape[0],) + k.shape[1:], np.float32)
    out[cols >= 0] = k[cols[cols >= 0]]
    return out


def din_forward(spec, W, feats, defect=None, row0=0):
    E, T = spec.emb_dim, spec.hist_len
    EP = 32 if E <= 32 else 64
    cand = O.numeric(feats, "movieId", np.float32).astype(np.int32)[:, 0]
    hist = np.concatenate([O.numeric(feats, k, np.float32) for k in O.din_history_keys(T)],
                          axis=1).astype(np.int32)
    tab = W["embedding"].astype(np.float32)
    H = np.zeros(hist.shape + (EP,), np.float32)
    H[..., :E] = tab[hist]
    C = np.zeros((cand.shape[0], EP), np.float32)
    C[:, :E] = tab[cand]
    au = W["au_dense/kernel"].astype(np.float32)
    w_sub, w_h, w_c, w_p = au[:E], au[E:2 * E], au[2 * E:3 * E], au[3 * E:]
    wh = _pad_rows(w_sub + w_h, EP).astype(np.float64)          # fp32 sums, as build_din uploads them
    wp = _pad_rows(w_p, EP).astype(np.float64)
    wc = _pad_rows(w_c - w_sub, EP).astype(np.float64)
    C64 = C.astype(np.float64)
    # activation unit: B operand W_r = fmaf(c, Wp, Wsub + Wh) per row, [B, EP, 32]
    Wr = (C64[:, :, None] * wp[None] + wh[None]).astype(np.float32)
    hit = _hit(defect, "au", H.shape, row0, pos_axis=1)
    D = split_product(H, Wr, AU_TERMS, "btk,bkj->btj", hit, defect.drop if hit is not None else None)
    z = D + (W["au_dense/bias"].astype(np.float64) + C64 @ wc)[:, None, :]
    a = O.prelu(z, W["au_prelu/alpha"].astype(np.float64))
    s = a @ W["au_out/kernel"].astype(np.float64)[:, 0] + np.float64(W["au_out/bias"][0])
    wgt = O.sigmoid(s)                                                        # [B, T]
    # pooling from the split tile
    hh, hl = split(H)
    phit = _hit(defect, "pool", H.shape, row0, pos_axis=1)
    if phit is not None:
        hl = np.where(phit, 0.0, hl)
    pooled = np.einsum("bt,btk->bk", wgt, hh + hl)
    # top MLP: X tile [userGenre1 | userId | pooled | candidate | movieGenre1] + numerics
    uid = O.identity_ids(feats, "userId", spec.n_users)
    ug = O.embedding_column(W["userGenre1_embedding"], O.genre_index(feats, "userGenre1"), np.float64)
    mg = O.embedding_column(W["movieGenre1_embedding"], O.genre_index(feats, "movieGenre1"), np.float64)
    u = O.embedding_column(W["userId_embedding"], uid, np.float64)
    X = np.zeros((cand.shape[0], 5 * EP))
    for b, part in enumerate((ug, u, pooled[:, :E], C64[:, :E], mg)):
        X[:, b * EP:b * EP + E] = part
    cols, num_rows = din_tile_columns(E, EP)
    k1 = W["dense/kernel"].astype(np.float32)
    W1 = _rows_of(k1, cols)
    if EP == 32:                     # on wgmma: the tile is fp32 in shared memory before its split
        h = _mlp_layer(X.astype(np.float32), W1, "mlp1", defect, row0)
    else:                            # CUDA cores, fp32: no split
        assert defect is None or defect.stage in ("au", "pool"), defect
        h = X @ W1.astype(np.float64)
    h = h + _numeric_term(feats, k1[num_rows], defect, row0) + W["dense/bias"].astype(np.float64)
    h = O.prelu(h, W["prelu/alpha"].astype(np.float64))
    k2 = W["dense_1/kernel"].astype(np.float32)
    h = _mlp_layer(h.astype(np.float32), k2, "mlp2", defect, row0) if EP == 32 else h @ k2.astype(np.float64)
    h = O.prelu(h + W["dense_1/bias"].astype(np.float64), W["prelu_1/alpha"].astype(np.float64))
    zl = h @ W["dense_2/kernel"].astype(np.float64) + W["dense_2/bias"].astype(np.float64)
    return O.sigmoid(zl), zl


# ---- embmlp_tc_kernel (EmbeddingMLP, Wide&Deep) ------------------------------------------------------
def embmlp_tile_columns(E):
    """Row of `dense/kernel` feeding each of embmlp_tc's 128 K columns (K = slot * 12 + e, slots
    movieGenre1..3, movieId, userGenre1..5, userId; -1 = zero), and the numerics' rows
    (csrc/placement.h place_embmlp)."""
    starts = [1 + k * E for k in range(3)] + [1 + 3 * E] + [5 + 4 * E + k * E for k in range(5)] + [5 + 9 * E]
    cols = np.full(128, -1, np.int64)
    for slot, s in enumerate(starts):
        cols[slot * 12:slot * 12 + E] = s + np.arange(E)
    nums = np.array([0, 1 + 4 * E, 2 + 4 * E, 3 + 4 * E, 4 + 4 * E, 5 + 10 * E, 6 + 10 * E])
    return cols, nums


def embmlp_forward(spec, W, feats, defect=None, row0=0):
    x = O._embmlp_input(spec, W, feats, np.float64)
    cols, num_rows = embmlp_tile_columns(spec.emb_dim)
    X = np.zeros((x.shape[0], 128))
    X[:, cols >= 0] = x[:, cols[cols >= 0]]
    k1 = W["dense/kernel"].astype(np.float32)
    h = _mlp_layer(X.astype(np.float32), _rows_of(k1, cols), "mlp1", defect, row0)
    h = np.maximum(h + _numeric_term(feats, k1[num_rows], defect, row0) + W["dense/bias"].astype(np.float64), 0)
    h = _mlp_layer(h.astype(np.float32), W["dense_1/kernel"].astype(np.float32), "mlp2", defect, row0)
    h = np.maximum(h + W["dense_1/bias"].astype(np.float64), 0)
    K = W["dense_2/kernel"].astype(np.float64)
    z = h @ K[:h.shape[1]] + W["dense_2/bias"].astype(np.float64)
    if spec.model == "widendeep":
        mid = O.identity_ids(feats, "movieId", spec.n_movies)
        rated = O.identity_ids(feats, "userRatedMovie1", spec.n_movies)
        z = z + K[h.shape[1] + O.crossed_bucket_array(mid, rated, spec.cross_buckets)]
    return O.sigmoid(z), z


# ---- deepfm_tc_kernel ----------------------------------------------------------------------------------
def deepfm_tile_columns(E):
    """Row of `dense/kernel` feeding each of deepfm_tc's 64 K columns ([deep movieId emb | deep userId emb],
    16 each, then zeros), and the numerics' rows (csrc/placement.h place_deepfm)."""
    cols = np.full(64, -1, np.int64)
    cols[:E] = 1 + np.arange(E)
    cols[16:16 + E] = 5 + E + np.arange(E)
    return cols, np.array([0, 1 + E, 2 + E, 3 + E, 4 + E, 5 + 2 * E, 6 + 2 * E])


def deepfm_forward(spec, W, feats, defect=None, row0=0):
    E = spec.emb_dim
    mid = O.identity_ids(feats, "movieId", spec.n_movies)
    uid = O.identity_ids(feats, "userId", spec.n_users)
    ig_i, ug_i = O.genre_index(feats, "movieGenre1"), O.genre_index(feats, "userGenre1")
    emb = lambda name, ids: O.embedding_column(W[name], ids, np.float64)
    item, user = emb("fm_movieId_embedding", mid), emb("fm_userId_embedding", uid)
    ig, ug = emb("fm_movieGenre1_embedding", ig_i), emb("fm_userGenre1_embedding", ug_i)
    dots = np.stack([(item * user).sum(1), (ig * ug).sum(1), (ig * user).sum(1), (item * ug).sum(1)], axis=1)
    X = np.zeros((mid.shape[0], 64))
    X[:, :E] = emb("deep_movieId_embedding", mid)
    X[:, 16:16 + E] = emb("deep_userId_embedding", uid)
    cols, num_rows = deepfm_tile_columns(E)
    k1 = W["dense/kernel"].astype(np.float32)
    h = _mlp_layer(X.astype(np.float32), _rows_of(k1, cols), "mlp1", defect, row0)
    h = np.maximum(h + _numeric_term(feats, k1[num_rows], defect, row0) + W["dense/bias"].astype(np.float64), 0)
    h = _mlp_layer(h.astype(np.float32), W["dense_1/kernel"].astype(np.float32), "mlp2", defect, row0)
    h = np.maximum(h + W["dense_1/bias"].astype(np.float64), 0)
    K = W["dense_2/kernel"].astype(np.float64)
    G, Vm = spec.n_genres, spec.n_movies
    o_mg, o_m, o_ug, o_u, o_d = 0, G, G + Vm, G + Vm + G, spec.fm1_width
    z = (O.indicator_weight(K[o_mg:o_m], ig_i, np.float64) + O.indicator_weight(K[o_m:o_ug], mid, np.float64)
         + O.indicator_weight(K[o_ug:o_u], ug_i, np.float64) + O.indicator_weight(K[o_u:o_d], uid, np.float64))
    z = z + dots @ K[o_d:o_d + 4] + h @ K[o_d + 4:] + W["dense_2/bias"].astype(np.float64)
    return O.sigmoid(z), z


FORWARD = {"din": din_forward, "embeddingmlp": embmlp_forward, "widendeep": embmlp_forward,
           "deepfm": deepfm_forward}


def forward(spec, W, feats, defect=None, batch_size=256):
    """float64 (prob[B,1], logit[B,1]) of the tensor-core kernel of `spec.model`, in row chunks of
    `batch_size` (the activation unit's operands are [rows, T, EP] per chunk)."""
    n = len(O._col(feats, "movieId"))
    ps, zs = [], []
    for lo in range(0, n, batch_size):
        sub = {k: np.asarray(v)[lo:lo + batch_size] for k, v in feats.items()}
        p, z = FORWARD[spec.model](spec, W, sub, defect, row0=lo)
        ps.append(p)
        zs.append(z)
    return np.concatenate(ps), np.concatenate(zs)
