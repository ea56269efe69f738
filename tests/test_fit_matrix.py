"""`model.fit` at every step-kernel instantiation, hidden depth and padding edge against the float64 training oracle.

NeuralCF's step is `ncf_train_step_kernel<EP, HP>` (EP in {12, 16, 32, 64}, HP in {16, 32}; csrc/ncf_train.cu) over
1 to 3 hidden layers; the trainer (csrc/trainer.cu) opts it into its three-layer dynamic shared memory at create,
which is above 48 KiB for some instantiations and covers every smaller shape.  DeepFM's is `deepfm_train_step_kernel<EP>`
(csrc/deepfm_train.cu), with the serving `deepfm_kernel<EP>` for validation and `Trainer.evaluate`; Wide&Deep's
`widendeep_train_step_kernel<EP>` with `embmlp_kernel<EP>`, DeepFM_v2's `deepfm2_train_step_kernel<EP>` with
`deepfm2_kernel<EP>`, and DIEN's `dien_train_step_kernel<EP>` (EP in {12, 16, 32}) with the `dien_kernel<EP, true>`
forward that `CTRModel.dien_evaluate` runs.  The trainer places its weights through the serving builders' placement
(csrc/placement.h) and gathers its exports back through it, and its step kernels restate the layout's offsets.  The defects such code invites - a padded column read as data, the last real column or unit dropped, the wrong
template, a tail tile mishandled - compound over a fit's steps.  `FIT_MATRIX` names one case per (model,
instantiation, width regime): the smallest E of a bucket, a partial pad and the exact bucket width, hidden width 1
and each model's limit, batches one row past the step's row tile or its double (64 rows for NeuralCF, 32 for the
others), about ten steps with the last batch partial, Keras's Adam and custom Adam, and per model one tiny vocabulary
whose ids repeat across the CTAs of every batch (the row-order dedupe of `table_grad_kernel`).  DIEN's cases also run
histories of 1, 2, an odd middle length and `kDienMaxT` positions, with padded positions (id 0) at the start, the
middle and the end of rows, one all-padding row and a candidate among its own history.

* GPU, per case: the trainer exports its initial weights bit for bit; the fit matches the float64 oracle within 4x
  (or the case's own multiple) the float32 oracle's own distance from it (plus one ulp); the step's forward is the
  serving forward, number for number; after the fit, the trainer's forward over its own padded arrays is that of a
  serving model rebuilt (with zero padding) from its exported weights; a second fit gives the same bits.
* CPU: `FIT_MATRIX` reaches every instantiation the launchers dispatch, 1, 2 and 3 hidden layers, width 1 and each
  model's limit, both sides of the shared-memory opt-in and its growth; each case's tolerance sees a dropped
  embedding column, a dropped hidden unit, a dropped batch row, the other Adam and each model's own defects; and the
  float64 oracle moves every tensor of every case, so that no dead unit leaves a chain untested.
"""
import collections
import functools
import glob
import os
import re

import numpy as np
import pytest

from oracle import deepfm_train, deepfm_v2_train, dien_train, ncf_train, widendeep_train
from sparrowrecsys_b200.spec import NUMERIC_KEYS, default_spec
from sparrowrecsys_b200.weights import init_aux_weights, init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc")
N_MOVIES, N_USERS = 1000, 1200          # the kernel matrix's small vocabularies; the golden ids are taken modulo them
SPREAD_MULTIPLE = 4.0                   # GPU-to-float64 distance allowed, in units of the float32-to-float64 distance
MAX_MULTIPLE = 8.0                      # no case may allow more
DEFECT_MULTIPLE = 10.0                  # a defect must move some tensor by this many tolerances
OPT_IN_BYTES = 48 * 1024                # dynamic shared memory a kernel gets without cudaFuncSetAttribute
TILE_ROWS = {"neuralcf": 64, "deepfm": 32, "widendeep": 32, "deepfm_v2": 32, "dien": 32}
# each hidden layer's widest width the trainer takes (csrc/trainer.cu check_shape); NeuralCF's 1 to 3 layers share one
MAX_HIDDEN = {"neuralcf": (32,), "deepfm": (64, 64), "widendeep": (128, 128), "deepfm_v2": (32, 16), "dien": (128, 64)}
HIDDEN_LAYERS = {"deepfm": ("dense", "dense_1"), "widendeep": ("dense", "dense_1"), "deepfm_v2": ("deep", "deep_1"),
                 "dien": ("dense", "dense_1")}
STEP_KERNEL = {"neuralcf": "ncf_train_step_kernel", "deepfm": "deepfm_train_step_kernel",
               "widendeep": "widendeep_train_step_kernel", "deepfm_v2": "deepfm2_train_step_kernel",
               "dien": "dien_train_step_kernel"}
# the forward of the trainer's validation and evaluate (DIEN: of `CTRModel.dien_evaluate`, dien_kernel<EP, true>)
FORWARD_KERNEL = {"deepfm": "deepfm_kernel", "widendeep": "embmlp_kernel", "deepfm_v2": "deepfm2_kernel",
                  "dien": "dien_kernel"}
ORACLE = {"neuralcf": ncf_train, "deepfm": deepfm_train, "widendeep": widendeep_train, "deepfm_v2": deepfm_v2_train,
          "dien": dien_train}
# the serving model whose forward each model's step and trainer forward share: (kernel name, options)
SERVING = {"neuralcf": ("ncf_kernel<neural_cf_model_1>", None), "deepfm": ("deepfm_kernel", {"deepfm_impl": "cudacore"}),
           "widendeep": ("embmlp_kernel<wide&deep>", {"embmlp_impl": "cudacore"}), "deepfm_v2": ("deepfm2_kernel", None),
           "dien": ("dien_kernel", None)}
ADAM = {"lr": 0.003, "beta_1": 0.8, "beta_2": 0.99, "epsilon": 1e-6}
ADAM_NO_MOMENTUM = {"lr": 0.002, "beta_1": 0.0, "beta_2": 0.95, "epsilon": 1e-5}

FitCase = collections.namedtuple("FitCase", "model over B n epochs seed adam multiple",
                                 defaults=(SPREAD_MULTIPLE,))


def _ncf(E, hidden, B, n, seed, adam=None, epochs=1, **vocab):
    return FitCase("neuralcf", dict(emb_dim=E, hidden=hidden, **vocab), B, n, epochs, seed, adam)


def _fm(E, hidden, B, n, seed, adam=None, epochs=1, **vocab):
    return FitCase("deepfm", dict(emb_dim=E, hidden=hidden, **vocab), B, n, epochs, seed, adam)


def _wd(E, hidden, B, n, seed, adam=None, epochs=1, multiple=SPREAD_MULTIPLE, **over):
    return FitCase("widendeep", dict(emb_dim=E, hidden=hidden, **over), B, n, epochs, seed, adam, multiple)


def _fm2(E, hidden, B, n, seed, adam=None, epochs=1, multiple=SPREAD_MULTIPLE, **over):
    return FitCase("deepfm_v2", dict(emb_dim=E, hidden=hidden, **over), B, n, epochs, seed, adam, multiple)


def _dien(E, T, hidden, B, n, seed, adam=None, epochs=1, multiple=SPREAD_MULTIPLE, **over):
    return FitCase("dien", dict(emb_dim=E, hist_len=T, hidden=hidden, **over), B, n, epochs, seed, adam, multiple)


TINY = dict(n_movies=3, n_users=5)      # every id repeats in every batch, across its CTAs

# NeuralCF's step shared memory per case (restated by `step_smem_bytes` below) is in the comment
FIT_MATRIX = [
    # ---- ncf_train_step_kernel<EP, HP>: every pair; hidden 1 / 16 / 17 / 32; 1, 2 and 3 layers ----
    _ncf(1, (1,), 65, 615, 0),                                   # <12, 16>   15.9 KiB
    _ncf(12, (17, 9), 129, 1231, 1, ADAM),                       # <12, 32>   45.6 KiB, just under the opt-in
    _ncf(13, (16, 16), 65, 300, 2, epochs=2),                    # <16, 16>   27.5 KiB
    _ncf(16, (32, 32, 32), 129, 1231, 3, ADAM),                  # <16, 32>   68.8 KiB
    _ncf(17, (1,), 65, 615, 4, ADAM_NO_MOMENTUM),                # <32, 16>   28.4 KiB
    _ncf(32, (17, 9), 65, 615, 5),                               # <32, 32>   60.6 KiB
    _ncf(32, (9, 32, 17), 129, 600, 6, ADAM, epochs=2),          # <32, 32>   80.8 KiB: the opt-in grows
    _ncf(33, (16, 16, 16), 65, 615, 7),                          # <64, 16>   66.5 KiB
    _ncf(64, (32, 32, 32), 129, 1231, 8, ADAM),                  # <64, 32>  104.8 KiB
    # measured on an H100 at 700 W: dense_2/bias lands 5.8x the float32 spread from float64, but that spread is
    # 0.3 ulp and the error 1.7 ulp, inside the rule's one-ulp term
    _ncf(64, (32, 17), 200, 1877, 9, ADAM, **TINY),              # <64, 32>   84.6 KiB, below the size opted in
    # ---- deepfm_train_step_kernel<EP> and deepfm_kernel<EP>: every EP; widths 1 and 64 ----
    _fm(1, (1, 1), 33, 314, 0),                                  # EP 12
    _fm(12, (64, 64), 65, 615, 1, ADAM),                         # EP 12
    _fm(13, (17, 33), 33, 314, 2, ADAM_NO_MOMENTUM),             # EP 16
    _fm(16, (37, 5), 33, 314, 3),                                # EP 16
    _fm(16, (64, 1), 65, 300, 4, ADAM, epochs=2),                # EP 16
    _fm(17, (1, 64), 33, 314, 5),                                # EP 32
    # measured on an H100 at 700 W: dense_2/bias lands 4.7x the float32 spread (0.27 ulp) from float64, at 1.3 ulp
    _fm(32, (63, 64), 65, 615, 6, ADAM),                         # EP 32
    _fm(33, (64, 1), 33, 314, 7, ADAM),                          # EP 64
    _fm(64, (37, 5), 65, 615, 8),                                # EP 64
    _fm(64, (64, 64), 97, 900, 9, ADAM, **TINY),                 # EP 64
    # ---- widendeep_train_step_kernel<EP> and embmlp_kernel<EP>: every EP; widths 1, 127 and 128; 1 and a prime
    # number of crossed buckets ----
    _wd(1, (1, 128), 33, 314, 0),                                # EP 12
    _wd(12, (128, 1), 65, 615, 1, ADAM, cross_buckets=1),        # EP 12
    _wd(13, (127, 127), 33, 314, 2, cross_buckets=7),            # EP 16
    _wd(16, (1, 1), 33, 150, 3, ADAM_NO_MOMENTUM, epochs=2),     # EP 16
    _wd(17, (128, 128), 65, 615, 4),                             # EP 32
    _wd(32, (17, 1), 33, 314, 5, ADAM, cross_buckets=1),         # EP 32
    _wd(33, (1, 1), 33, 314, 6, cross_buckets=97),               # EP 64, the partial pad
    _wd(64, (127, 1), 33, 314, 7, ADAM),                         # EP 64
    _wd(64, (128, 127), 97, 900, 8, ADAM, cross_buckets=7, **TINY),  # EP 64
    # ---- deepfm2_train_step_kernel<EP> and deepfm2_kernel<EP>: every EP; widths 1, 31, 32 and 1, 15, 16 ----
    _fm2(1, (32, 16), 33, 314, 0),                               # EP 12
    # measured on an H100 at 700 W: first_cat/bias lands 11.6x the float32 spread from float64, at 6.9e-9 (1.8 ulp)
    # against 5.9e-10; the float32 oracle with each batch's rows reversed lands 7.3x from it
    _fm2(12, (1, 16), 65, 615, 1, ADAM, multiple=6.0),           # EP 12
    _fm2(13, (31, 15), 33, 314, 2, ADAM_NO_MOMENTUM),            # EP 16
    _fm2(16, (32, 1), 33, 150, 3, epochs=2),                     # EP 16
    _fm2(17, (1, 1), 33, 314, 4, ADAM),                          # EP 32
    _fm2(32, (31, 16), 65, 615, 5),                              # EP 32
    _fm2(33, (1, 15), 33, 314, 6, ADAM),                         # EP 64, the partial pad
    _fm2(64, (31, 1), 65, 615, 7, ADAM_NO_MOMENTUM),             # EP 64
    _fm2(64, (32, 16), 97, 900, 8, **TINY),                      # EP 64
    # ---- dien_train_step_kernel<EP> and dien_kernel<EP, true>: every EP; widths 1, 127, 128 and 1, 63, 64;
    # histories of 1, 2, odd and kDienMaxT positions ----
    _dien(1, 2, (128, 64), 33, 314, 0),                          # EP 12
    # measured on an H100 at 700 W: dense_2/bias lands 5.2x the float32 spread, at 3.1e-9 (under one ulp).  At seed 1
    # att_out/bias landed 37x (2.1 ulp), but there the float32 oracle with each batch's rows reversed lands 145x from
    # float64, so seed 16 is one whose float32 spread is no lucky near miss
    _dien(12, 64, (1, 1), 33, 314, 16, ADAM, multiple=6.0),      # EP 12
    _dien(12, 1, (127, 63), 65, 615, 2),                         # EP 12
    _dien(13, 1, (127, 63), 33, 314, 3, ADAM_NO_MOMENTUM),       # EP 16
    _dien(16, 9, (1, 64), 97, 900, 4, ADAM, **TINY),             # EP 16
    # measured on an H100 at 700 W: dense/kernel lands 5.1x the float32 spread, 1.42e-6 against 2.81e-7; the float32
    # oracle with each batch's rows reversed lands 3.4x from it
    _dien(16, 64, (128, 63), 33, 314, 8, multiple=6.0),          # EP 16
    # measured on an H100 at 700 W: att_out/bias lands 11.2x the float32 spread, at 8.2e-9 (2.2 ulp) against 7.3e-10;
    # the float32 oracle with each batch's rows reversed lands 6.1x from it
    _dien(17, 33, (127, 1), 33, 150, 5, epochs=2, multiple=8.0),  # EP 32
    # measured on an H100 at 700 W: userGenre1_embedding lands 8.15x the float32 spread, 1.019e-6 against 1.25e-7,
    # inside 8x only by the one-ulp term (3e-8); reversing each batch's rows does not move the float32 oracle's
    # distance on this tensor, so whether an order of the sums accounts for it is not shown
    _dien(32, 64, (128, 64), 65, 615, 6, ADAM, multiple=8.0),    # EP 32
    _dien(32, 2, (1, 63), 33, 314, 7),                           # EP 32
]


def _adam_id(adam):
    return "keras" if adam is None else "b1_0" if adam["beta_1"] == 0 else "adam"


def _case_id(c):
    parts = [c.model, "E%d" % c.over["emb_dim"]]
    if "hist_len" in c.over:
        parts.append("T%d" % c.over["hist_len"])
    parts += ["h" + "x".join(map(str, c.over["hidden"])), "B%d" % c.B, "n%d" % c.n]
    if c.epochs != 1:
        parts.append("ep%d" % c.epochs)
    if "n_movies" in c.over:
        parts.append("V%dx%d" % (c.over["n_movies"], c.over["n_users"]))
    if "cross_buckets" in c.over:
        parts.append("cb%d" % c.over["cross_buckets"])
    parts += [_adam_id(c.adam), "s%d" % c.seed]
    return "-".join(parts)


def _spec(c):
    return default_spec(c.model, **dict(dict(n_movies=N_MOVIES, n_users=N_USERS), **c.over))


def _steps(c):
    return c.epochs * -(-c.n // c.B)


def round_ep(E):
    """The trainer's padded embedding width (srs_trainer_create; csrc/model.cu round_ep)."""
    return 12 if E <= 12 else 16 if E <= 16 else 32 if E <= 32 else 64


def instantiations(c):
    """The step (and forward) kernel instantiations a case runs, by srs_trainer_create's rule: EP from E; NeuralCF's
    HP = 16 if its widest hidden layer is at most 16, else 32; the other models pad every hidden layer to their
    limit."""
    spec = _spec(c)
    EP = round_ep(spec.emb_dim)
    if c.model == "neuralcf":
        return {(STEP_KERNEL[c.model], EP, 16 if max(spec.hidden) <= 16 else 32)}
    return {(STEP_KERNEL[c.model], EP), (FORWARD_KERNEL[c.model], EP) + (("true",) if c.model == "dien" else ())}


def _switch_cases(src, signature, launch):
    """The EPs of the `case N: return <launch><N...>` lines in the body of the launcher whose definition starts with
    `signature`."""
    body = re.search(re.escape(signature) + r".*?\n}", src, re.S)
    return [int(ep) for ep in re.findall(r"case (\d+): return %s<\1\b" % re.escape(launch), body.group(0))] \
        if body else []


def dispatched_instantiations():
    """Every instantiation the trainer's launchers in csrc/*.cu can dispatch, read from their dispatch lines: the step
    kernels' cases, and the cases of the switches of `launch_deepfm`, `launch_embmlp`, `launch_deepfm2` and
    `launch_dien_aux` (the forwards of the trainer's validation and evaluate, and of `CTRModel.dien_evaluate`)."""
    found = set()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        with open(path) as f:
            src = f.read()
        for ep, hp in re.findall(r"SRS_TRAIN_CASE\((\d+), (\d+)\)", src):
            found.add(("ncf_train_step_kernel", int(ep), int(hp)))
        for macro, kernel in (("SRS_DEEPFM_TRAIN_CASE", "deepfm_train_step_kernel"),
                              ("SRS_WD_STEP_CASE", "widendeep_train_step_kernel"),
                              ("SRS_FM2_STEP_CASE", "deepfm2_train_step_kernel"),
                              ("SRS_DIEN_STEP_CASE", "dien_train_step_kernel")):
            for ep in re.findall(r"%s\((\d+)\)" % macro, src):
                found.add((kernel, int(ep)))
        for signature, launch, kernel in (
                ("cudaError_t launch_deepfm(const DeepFmParams& p", "launch_deepfm_t", ("deepfm_kernel",)),
                ("cudaError_t launch_embmlp(const EmbMlpParams& p", "launch_embmlp_t", ("embmlp_kernel",)),
                ("cudaError_t launch_deepfm2(const DeepFm2Params& p", "launch_deepfm2_t", ("deepfm2_kernel",))):
            for ep in _switch_cases(src, signature, launch):
                found.add(kernel[:1] + (ep,))
        body = re.search(r"cudaError_t launch_dien_aux\(const DienParams& p.*?\n}", src, re.S)
        if body:
            for ep in re.findall(r"case (\d+): return launch_dien_t<\1, true>", body.group(0)):
                found.add(("dien_kernel", int(ep), "true"))
    return found


def dien_max_hist_len():
    """csrc/kernels.h kDienMaxT: the longest history DIEN's step trains."""
    with open(os.path.join(CSRC, "kernels.h")) as f:
        return int(re.search(r"constexpr int kDienMaxT = (\d+);", f.read()).group(1))


def step_smem_bytes(c):
    """csrc/ncf_train.cu step_smem_bytes: build_ncf's blob (each hidden layer's kernel [2EP or HP][HP] and bias [HP],
    then the output's [HP] and [4]) and, per row of the 64-row CTA, x [2EP], each layer's output and delta [HP] and
    dL/dz."""
    spec = _spec(c)
    EP, HP, L = round_ep(spec.emb_dim), 16 if max(spec.hidden) <= 16 else 32, len(spec.hidden)
    blob = sum((2 * EP if l == 0 else HP) * HP + HP for l in range(L)) + HP + 4
    return 4 * (blob + TILE_ROWS["neuralcf"] * (2 * EP + 2 * L * HP + 1))


# ---- the inputs and the oracle's fits ------------------------------------------------------------------
def _per_case(fn):
    """fn(case) computed once per case id (a case holds dicts, so it is not hashable itself)."""
    memo = {}

    @functools.wraps(fn)
    def once(case):
        key = _case_id(case)
        if key not in memo:
            memo[key] = fn(case)
        return memo[key]
    return once


@functools.lru_cache(maxsize=None)
def _trainset(model):
    return dict(np.load(os.path.join(GOLDEN, "%s_trainset.npz" % model)))


def _fm_rows(ts, n):
    """n DeepFM rows: the training set's first three rows without a userGenre1 first (as test_gpu_fit_deepfm.py's
    `_rows`), then the next rows in file order; rows 1 and 40 lose their movieGenre1 (the set has none missing)."""
    missing = np.flatnonzero(ts["userGenre1"] < 0)
    rest = np.setdiff1d(np.arange(n + 3), missing[:3])[: n - 3]
    idx = np.concatenate([missing[:3], rest])
    f = {k: np.ascontiguousarray(v[idx]) for k, v in ts.items()}
    f["movieGenre1"] = f["movieGenre1"].astype(np.int32)
    f["movieGenre1"][[1, 40]] = -1
    return f


def _unit_numerics(rng, n):
    """The 7 numerics at unit scale.  The data's raw scale (release years near 1995, rating counts in the thousands)
    puts every row on one side of a narrow layer's relu, and a unit that is dead on every row hides its chain."""
    return {k: rng.normal(0.0, 1.0, n).astype(np.float32) for k in NUMERIC_KEYS}


def _wd_rows(spec, n, seed):
    """n Wide&Deep rows over the spec's vocabularies: each genre slot missing on about one row in twenty, every slot
    missing on row 0, and rows 1 and 2 on one crossed bucket."""
    rng = np.random.default_rng(seed)
    f = {"movieId": rng.integers(0, spec.n_movies, n).astype(np.int32),
         "userId": rng.integers(0, spec.n_users, n).astype(np.int32),
         "userRatedMovie1": rng.integers(0, spec.n_movies, n).astype(np.int32),
         "label": rng.integers(0, 2, n).astype(np.int32)}
    for key in ["movieGenre%d" % k for k in (1, 2, 3)] + ["userGenre%d" % k for k in (1, 2, 3, 4, 5)]:
        f[key] = rng.integers(-1, spec.n_genres, n).astype(np.int8)
        f[key][0] = -1
    f["movieId"][2], f["userRatedMovie1"][2] = f["movieId"][1], f["userRatedMovie1"][1]
    f.update(_unit_numerics(rng, n))
    return f


def _fm2_rows(spec, n, seed):
    """n DeepFM_v2 rows over the spec's vocabularies: each genre field missing on about one row in twenty, both on
    rows 0 and 5."""
    rng = np.random.default_rng(seed)
    f = {"movieId": rng.integers(0, spec.n_movies, n).astype(np.int32),
         "userId": rng.integers(0, spec.n_users, n).astype(np.int32),
         "label": rng.integers(0, 2, n).astype(np.int32)}
    for key in ("movieGenre1", "userGenre1"):
        f[key] = rng.integers(-1, spec.n_genres, n).astype(np.int8)
        f[key][[0, 5]] = -1
    f.update(_unit_numerics(rng, n))
    return f


def _dien_weights(spec, seed):
    """The initialisers of the model and its auxiliary head, with every bias and PReLU alpha non-zero."""
    W = {**init_weights(spec, seed), **init_aux_weights(spec, seed)}
    rng = np.random.default_rng(seed + 50)
    for k in W:
        if k.endswith("/bias") or k.endswith("/alpha"):
            W[k] = rng.uniform(-0.3, 0.3, size=W[k].shape).astype(np.float32)
    return W


def _dien_rows(spec, n, seed):
    """n DIEN rows with negatives and labels: histories padded (id 0) at the start, the middle and the end of rows
    besides the generator's padded tails, row 5 all padding, row 4's candidate its own first history id, missing
    genres on every seventh row."""
    from sparrowrecsys_b200.features import negative_history, synthetic_features
    from oracle.ctr_oracle import din_history_keys
    f = synthetic_features(spec, n, seed=seed)
    keys = din_history_keys(spec.hist_len)
    for k in keys:
        f[k] = np.array(f[k])
    for i in range(n):
        if i % 4 and spec.hist_len > 1:
            f[keys[(0, len(keys) // 2, -1)[i % 4 - 1]]][i] = 0
    for k in keys:
        f[k][5] = 0
    f["movieId"] = np.array(f["movieId"])
    f["movieId"][4] = f[keys[0]][4]                # the generator never pads position 0
    for g in ("movieGenre1", "userGenre1"):
        f[g] = np.array(f[g], dtype=object)
        f[g][::7] = ""
    f.update(negative_history(f, spec.hist_len, seed, n_movies=spec.n_movies))
    rng = np.random.default_rng(seed)
    f.update(_unit_numerics(rng, n))
    f["label"] = (rng.random(n) < 0.5).astype(np.int32)
    return f


@_per_case
def _inputs(c):
    """(W0, rows, orders) of a case: the reference initialisers with test biases at the case's seed; the golden
    training rows with their ids taken modulo the case's vocabularies (NeuralCF, DeepFM) or rows drawn at the
    case's seed (the others); one permutation per epoch."""
    spec = _spec(c)
    W0 = _dien_weights(spec, c.seed) if c.model == "dien" else init_weights(spec, c.seed, for_test=True)
    if c.model in ("neuralcf", "deepfm"):
        ts = _trainset(c.model)
        if c.model == "neuralcf":
            f = {k: np.ascontiguousarray(ts[k][:c.n]) for k in ("movieId", "userId", "label")}
        else:
            f = _fm_rows(ts, c.n)
        f["movieId"] = (f["movieId"] % spec.n_movies).astype(np.int32)
        f["userId"] = (f["userId"] % spec.n_users).astype(np.int32)
    else:
        f = {"widendeep": _wd_rows, "deepfm_v2": _fm2_rows, "dien": _dien_rows}[c.model](spec, c.n, c.seed)
    return W0, f, ncf_train.epoch_orders(c.n, c.epochs, 11)


@_per_case
def _rows(c):
    """The oracle's row object of a case's rows (NeuralCF reads the id columns directly)."""
    f = _inputs(c)[1]
    if c.model == "dien":
        return dien_train.Rows.from_features(f, c.over["hist_len"])
    return {"deepfm": deepfm_train.Rows, "widendeep": widendeep_train.Rows,
            "deepfm_v2": deepfm_v2_train.Rows}[c.model].from_features(f)


def _oracle_fit(c, dtype, adam):
    W0, f, orders = _inputs(c)
    if c.model == "neuralcf":
        return ncf_train.fit(W0, f["movieId"], f["userId"], f["label"], orders, c.B, dtype, hp=adam)[0]
    if c.model == "dien":
        return dien_train.fit(W0, _rows(c), orders, c.B, dtype, hp=adam)[0]
    return ORACLE[c.model].fit(W0, _rows(c), f["label"], orders, c.B, dtype, hp=adam)[0]


@_per_case
def _oracle(c):
    """(W64, W32, tolerance per tensor): the case's fit at float64 and float32, and the GPU's allowance, the case's
    multiple (4x unless measured otherwise) of the float32 fit's distance from the float64 one plus one float32 ulp
    of the tensor's largest value (no float32 result is nearer than that)."""
    W64, W32 = _oracle_fit(c, np.float64, c.adam), _oracle_fit(c, np.float32, c.adam)
    tol = {k: c.multiple * float(np.abs(W32[k] - W64[k]).max())
           + float(np.spacing(np.float32(np.abs(W64[k]).max()))) for k in W64}
    return W64, W32, tol


def _distance(Wa, Wb, tol):
    """(the largest distance in tolerances over the tensors, its tensor)."""
    return max((float(np.abs(Wa[k] - Wb[k]).max()) / tol[k], k) for k in tol)


# ---- CPU: the matrix is complete, and its tolerances see the defects -------------------------------------
def test_matrix_reaches_every_step_and_forward_instantiation():
    """Every step-kernel instantiation the trainer dispatches, and every instantiation of the serving forwards the
    trainer and `CTRModel.dien_evaluate` share with the steps, is run by some FIT_MATRIX case."""
    dispatched = dispatched_instantiations()
    assert {d[0] for d in dispatched} == {"ncf_train_step_kernel", "deepfm_train_step_kernel", "deepfm_kernel",
                                          "widendeep_train_step_kernel", "embmlp_kernel",
                                          "deepfm2_train_step_kernel", "deepfm2_kernel",
                                          "dien_train_step_kernel", "dien_kernel"}, dispatched
    reached = set().union(*(instantiations(c) for c in FIT_MATRIX))
    missing = sorted(dispatched - reached)
    assert not missing, "no FIT_MATRIX case runs %s" % ", ".join("%s<%s>" % (d[0], ", ".join(map(str, d[1:])))
                                                                 for d in missing)


def test_matrix_covers_depths_widths_and_batches():
    dispatched = dispatched_instantiations()
    for model in TILE_ROWS:
        cases = [c for c in FIT_MATRIX if c.model == model]
        assert cases, model
        if model == "neuralcf":
            widths = {h for c in cases for h in c.over["hidden"]}
            assert {1, MAX_HIDDEN[model][0]} <= widths, (model, widths)
        else:                                  # width 1 and the limit in each layer, and one below the limit
            for layer, limit in enumerate(MAX_HIDDEN[model]):
                widths = {c.over["hidden"][layer] for c in cases}
                edges = {1, limit} if model == "deepfm" else {1, limit - 1, limit}
                assert edges <= widths, (model, layer, widths)
        # the smallest E of each EP bucket the model's step dispatches, a partial pad and the exact width
        eps = {d[1] for d in dispatched if d[0] == STEP_KERNEL[model]}
        Es = {c.over["emb_dim"] for c in cases}
        want = {E for E in (1, 12, 13, 16, 17, 32, 33, 64) if round_ep(E) in eps}
        assert want <= Es, (model, sorted(want - Es))
        assert any(_spec(c).n_movies <= 3 and _spec(c).n_users <= 5 and c.B > 2 * TILE_ROWS[model] for c in cases), \
            "%s: no case whose ids repeat across the CTAs of a batch" % model
        for c in cases:
            tile = TILE_ROWS[model]
            assert c.B > tile and c.B % tile != 0, (_case_id(c), "the batch must straddle the row tile")
            assert c.n % c.B != 0, (_case_id(c), "the last batch must be partial")
            assert 8 <= _steps(c) <= 12, (_case_id(c), _steps(c))
            assert SPREAD_MULTIPLE <= c.multiple <= MAX_MULTIPLE, (_case_id(c), c.multiple)
        adams = [_adam_id(c.adam) for c in cases]
        assert "b1_0" in adams and "adam" in adams and 0.3 <= adams.count("keras") / len(adams) <= 0.7, (model, adams)
        assert any(c.epochs == 2 for c in cases), model
    assert {len(c.over["hidden"]) for c in FIT_MATRIX if c.model == "neuralcf"} == {1, 2, 3}
    buckets = {_spec(c).cross_buckets for c in FIT_MATRIX if c.model == "widendeep"}
    assert 1 in buckets and any(b > 2 and all(b % d for d in range(2, b)) for b in buckets), buckets
    Ts = {c.over["hist_len"] for c in FIT_MATRIX if c.model == "dien"}
    assert {1, 2, dien_max_hist_len()} <= Ts and any(t % 2 and 2 < t < dien_max_hist_len() for t in Ts), Ts


def test_dien_rows_reach_the_padding_edges():
    """Each DIEN case's rows pad (id 0) the first, a middle and the last history position of some rows (where T
    allows), hold one all-padding row, a candidate among its own history, and rows without a genre."""
    for c in FIT_MATRIX:
        if c.model != "dien":
            continue
        r, T = _rows(c), c.over["hist_len"]
        pad = r.hist == 0
        assert pad.all(1).any() and (~pad).any(1).any(), _case_id(c)
        for t in ({0, T // 2, T - 1} if T > 1 else ()):
            assert (pad[:, t] & (~pad).any(1)).any(), (_case_id(c), t)
        assert any(r.mid[i] in r.hist[i] for i in range(c.n)), _case_id(c)
        assert (r.ig < 0).any() and (r.ug < 0).any(), _case_id(c)


def test_matrix_crosses_the_shared_memory_opt_in_and_grows_it():
    """`srs_trainer_create` opts a NeuralCF instantiation in once, at its three-layer shared memory: cases on both
    sides of 48 KiB, and an instantiation run at a shape that is followed (in the order the GPU tests run) by a larger
    one, so that the create-time opt-in at the largest size covers each smaller shape."""
    ncf = [c for c in FIT_MATRIX if c.model == "neuralcf"]
    smem = [step_smem_bytes(c) for c in ncf]
    assert any(s <= OPT_IN_BYTES for s in smem) and any(s > OPT_IN_BYTES for s in smem), smem
    assert max(smem) <= 227 * 1024, smem                      # an H100 CTA's dynamic shared memory limit
    grows = [(i, j) for i in range(len(ncf)) for j in range(i + 1, len(ncf))
             if instantiations(ncf[i]) == instantiations(ncf[j]) and OPT_IN_BYTES < smem[i] < smem[j]]
    assert grows, "no instantiation is opted in and then asked for more"


def test_matrix_cases_are_distinct():
    ids = [_case_id(c) for c in FIT_MATRIX]
    assert len(ids) == len(set(ids))


def _still(case):
    """The tensors a case's fit leaves untrained by construction: DIEN's `augru_h0` (not a variable), and at T = 1
    (no position t >= 1) its recurrent kernel, which only multiplies the zero initial state, and its auxiliary
    head."""
    if case.model != "dien":
        return set()
    still = {"augru_h0"}
    if case.over["hist_len"] == 1:
        still |= {"gru_recurrent/kernel"} | {"aux_%s_%s/%s" % (side, layer, p) for side in ("pos", "neg")
                                             for layer in ("dense", "out") for p in ("kernel", "bias")}
    return still


@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_float64_oracle_moves_every_tensor(case):
    """A unit that is dead on every row of every batch leaves its chain without a gradient, and then a GPU fit that
    lost that chain would pass; each case's seed and rows are chosen so that every tensor moves by many tolerances."""
    W0 = _inputs(case)[0]
    W64, _, tol = _oracle(case)
    still = _still(case)
    for k in W0:
        moved = float(np.abs(W64[k] - W0[k]).max())
        if k in still:
            assert moved == 0, (k, moved)
        else:
            assert moved > DEFECT_MULTIPLE * tol[k], (k, moved, tol[k])


def _defects(case):
    """(name, gradients function, Adam) of the defects a trainer could have, each injected through the module
    global `gradients` that the oracle's `fit` calls."""
    model = case.model
    intact = ORACLE[model].gradients
    E, hidden = case.over["emb_dim"], case.over["hidden"]
    layers = ["dense_%d" % l for l in range(len(hidden))] if model == "neuralcf" else HIDDEN_LAYERS[model]

    def edited(edit):
        def grads(W, *args):
            out = intact(W, *args)
            edit(out[0], W, *args, out=out)
            return out
        return grads

    def column(g, *_, out):
        for k in g:
            if k.endswith("embedding"):
                g[k][:, E - 1] = 0

    def unit(g, *_, out):
        for l, (layer, h) in enumerate(zip(layers, hidden)):
            g[layer + "/kernel"][:, h - 1] = 0
            g[layer + "/bias"].reshape(-1)[h - 1] = 0
            if model == "dien":
                g[("prelu/alpha", "prelu_1/alpha")[l]][h - 1] = 0

    def last_row(W, *args):
        # NeuralCF: (mid, uid, y, dtype); DeepFM, Wide&Deep, DeepFM_v2: (rows, y, dtype); DIEN: (rows, y, dtype,
        # defect)
        n_cols = 3 if model == "neuralcf" else 2
        cols, rest = args[:n_cols], args[n_cols:]
        out = intact(W, *args)
        B = len(cols[-1])
        if B > 1:
            head = [a[:-1] for a in cols] if model == "neuralcf" else [cols[0].take(np.arange(B - 1)), cols[1][:-1]]
            g = intact(W, *head, *rest)[0]
            if model != "dien":                # a mean over the batch; DIEN's objective is a sum
                g = {k: v * ((B - 1) / B) for k, v in g.items()}
            out = (g,) + tuple(out[1:])
        return out

    def wide(g, W, r, y, dtype, out):          # the last row's crossed-bucket entry of dense_2/kernel
        p = out[1]
        hw = W["dense_1/kernel"].shape[1]
        b = r.bucket(widendeep_train.cross_buckets(W))[-1]
        g["dense_2/kernel"][hw + b, 0] -= (p[-1] - dtype(y[-1])) / dtype(len(y))

    def onehot(g, W, r, y, dtype, out):        # the last row's four one-hot entries of first_cat/kernel
        p = out[1]
        dfirst = (p[-1] - dtype(y[-1])) / dtype(len(y)) * dtype(W["out/kernel"][0, 0])
        for s in deepfm_v2_train.first_order_index(W, r)[:, -1]:
            if s >= 0:
                g["first_cat/kernel"][s, 0] -= dfirst

    yield "embedding column %d gets no gradient" % (E - 1), edited(column), case.adam
    yield "the last unit of each hidden layer gets no gradient", edited(unit), case.adam
    yield "the last row of each batch is left out", last_row, case.adam
    yield "the other Adam", intact, ADAM if case.adam is None else None
    if model == "widendeep":
        yield "the last row's wide entry is dropped", edited(wide), case.adam
    if model == "deepfm_v2":
        yield "the last row's one-hot entries are dropped", edited(onehot), case.adam
    if model == "dien":
        T = case.over["hist_len"]
        mutants = ["mean", "h0", "last"] + (["mask"] if (_rows(case).hist == 0).any() else []) + \
            (["aux", "step"] if T >= 2 else [])
        for d in mutants:
            yield "the oracle's mutant %r" % d, \
                functools.partial(lambda d, W, r, y, dtype=np.float32, defect=None: intact(W, r, y, dtype, d), d), \
                case.adam


@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_tolerance_sees_each_defect(case):
    """Each defect moves some tensor of the float64 fit by more than 10x the parity tolerance of the GPU test."""
    mod = ORACLE[case.model]
    W64, _, tol = _oracle(case)
    intact = mod.gradients
    for name, grads, adam in _defects(case):
        mod.gradients = grads
        try:
            Wd = _oracle_fit(case, np.float64, adam)
        finally:
            mod.gradients = intact
        far, k = _distance(Wd, W64, tol)
        assert far > DEFECT_MULTIPLE, "%s moves %s by only %.3g tolerances" % (name, k, far)


# ---- GPU: every case against the float64 oracle ------------------------------------------------------
def _trainer(case, W):
    from sparrowrecsys_b200.training import Trainer
    return Trainer(_spec(case), W, adam=case.adam)


def _serving(case, W):
    """The CUDA-core serving model of W, whose forward the step and the trainer's evaluate share."""
    from sparrowrecsys_b200.model import CTRModel
    name, options = SERVING[case.model]
    m = CTRModel(_spec(case), W, options=options)
    assert m.kernel_name == name
    return m


def _same_result(r, s):
    assert (r.rows, r.positives, r.correct) == (s.rows, s.positives, s.correct)
    assert (r.loss, r.accuracy, r.roc_auc, r.pr_auc) == (s.loss, s.accuracy, s.roc_auc, s.pr_auc)


def _one_step_in_file_order(tr, case, f):
    """The history of one step over all n rows in file order: the step's forward before its update."""
    return tr.fit(f, epochs=1, batch_size=case.n, order=[np.arange(case.n)])


@pytest.mark.gpu
@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_trainer_exports_its_initial_weights_exactly(case):
    W0 = _inputs(case)[0]
    with _trainer(case, W0) as tr:
        W = tr.weights()
        assert tr.iterations == 0
    assert W.keys() == W0.keys()
    for k in W0:
        assert W[k].shape == W0[k].shape and np.array_equal(W[k], W0[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_fit_matches_float64_oracle(case):
    """Every tensor within the case's multiple of the float32 oracle's spread (plus one ulp) of the float64 fit, and
    DIEN's augru_h0 bit for bit.  The test runs the cases in FIT_MATRIX's order in one process, so NeuralCF's <32, 32>
    opts in at 60.6 KiB and then grows to 80.8 KiB."""
    W0, f, orders = _inputs(case)
    W64, W32, tol = _oracle(case)
    with _trainer(case, W0) as tr:
        tr.fit(f, epochs=case.epochs, batch_size=case.B, order=orders)
        assert tr.iterations == _steps(case)
        Wg = tr.weights()
    if case.model == "dien":
        assert np.array_equal(Wg["augru_h0"], W0["augru_h0"])
    ratios = {}
    for k in W0:
        assert Wg[k].shape == W0[k].shape, k
        spread = float(np.abs(W32[k] - W64[k]).max())
        err = float(np.abs(Wg[k].astype(np.float64) - W64[k]).max())
        ratios[k] = err / spread if spread else float("inf") if err else 0.0
        assert err <= tol[k], (k, err, spread, tol[k])
    k = max(ratios, key=ratios.get)
    ulp = float(np.spacing(np.float32(np.abs(W64[k]).max())))
    print("%s: largest GPU error / float32 spread %.2f (%s: error %.3g, spread %.3g, ulp %.3g)"
          % (_case_id(case), ratios[k], k, ratios[k] * float(np.abs(W32[k] - W64[k]).max()),
             float(np.abs(W32[k] - W64[k]).max()), ulp))


@pytest.mark.gpu
@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_step_forward_is_the_serving_forward(case):
    """One step over all n rows in file order: its history (the step's outputs before its update) is the serving
    model's evaluate of the same rows in one batch, number for number (DIEN: `dien_evaluate`)."""
    W0, f, _ = _inputs(case)
    with _trainer(case, W0) as tr:
        h = _one_step_in_file_order(tr, case, f)
    with _serving(case, W0) as m:
        if case.model == "dien":
            assert h == {k: [v] for k, v in m.dien_evaluate(f).items()}
        else:
            loss, acc, roc, pr = m.evaluate(f, batch_size=case.n)
            assert (h["loss"][0], h["accuracy"][0], h["auc"][0], h["auc_1"][0]) == (loss, acc, roc, pr)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_padding_stays_zero(case):
    """After the fit, the trainer's forward over its own padded arrays (through the parameters it keeps over them) is
    the forward of a serving model built from the exported weights, whose padding is zero by construction: its
    evaluate, or for DIEN, which has no trainer evaluate, the history of one more step over all rows in file
    order against `dien_evaluate`."""
    W0, f, orders = _inputs(case)
    with _trainer(case, W0) as tr:
        tr.fit(f, epochs=case.epochs, batch_size=case.B, order=orders)
        W = tr.weights()
        if case.model == "dien":
            got = _one_step_in_file_order(tr, case, f)
        else:
            got = tr.evaluate_result(f)
    with _serving(case, W) as m:
        if case.model == "dien":
            assert got == {k: [v] for k, v in m.dien_evaluate(f).items()}
        else:
            _same_result(got, m.evaluate_result(f, batch_size=case.n))
            assert got.rows == case.n


@pytest.mark.gpu
@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_fit_is_deterministic(case):
    W0, f, orders = _inputs(case)
    outs = []
    for _ in range(2):
        with _trainer(case, W0) as tr:
            outs.append((tr.fit(f, epochs=case.epochs, batch_size=case.B, order=orders), tr.weights()))
    assert outs[0][0] == outs[1][0]
    for k in W0:
        assert np.array_equal(outs[0][1][k], outs[1][1][k]), k
