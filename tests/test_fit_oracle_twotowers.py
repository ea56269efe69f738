"""CPU checks of the two-tower model's `fit` (neural_cf_model_2 with its final Dense; DESIGN.md section 4.27): its
float64 oracle (oracle/twotowers_train.py) against central differences and Keras Adam's known answers, the golden
fixture, the trainer ABI's rejections that need no device, the step kernel's dispatch lines against the GPU matrix
(`TT_MATRIX`, run by tests/test_gpu_fit_twotowers.py), and that each matrix case's parity tolerance sees the defects
a step could have.

`TT_MATRIX` names one case per (instantiation, width regime) of `twotowers_train_step_kernel<EP, HP>` (EP in
{12, 16, 32, 64}, HP in {16, 32}; csrc/twotowers_train.cu) over 1 to 3 hidden layers per tower: the smallest E of a
bucket, a partial pad and the exact bucket width, hidden widths 1, 16, 17 and 32, step shared memory on both sides of
48 KiB and one instantiation run at a shape below a later, larger one (the trainer opts in once, at its three-layer
size), batches of 65, 129 and 200 rows (one past the 64-row CTA or its double), about ten steps with the last batch
partial, Keras's Adam and custom Adam (beta_1 = 0 included), and a 3-movie, 5-user vocabulary whose ids repeat
across the CTAs of every batch.
"""
import collections
import ctypes as C
import functools
import glob
import json
import os
import re

import numpy as np
import pytest

from oracle import ctr_oracle, ncf_train, twotowers_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc")
N_MOVIES, N_USERS = 1000, 1200          # the matrix's small vocabularies; the golden ids are taken modulo them
SPREAD_MULTIPLE = 4.0                   # GPU-to-float64 distance allowed, in units of the float32-to-float64 distance
DEFECT_MULTIPLE = 10.0                  # a defect must move some tensor by this many tolerances
OPT_IN_BYTES = 48 * 1024                # dynamic shared memory a kernel gets without cudaFuncSetAttribute
SMEM_LIMIT = 227 * 1024                 # an H100 CTA's dynamic shared memory limit
TILE_ROWS = 64                          # rows per CTA of the step
ADAM = {"lr": 0.003, "beta_1": 0.8, "beta_2": 0.99, "epsilon": 1e-6}
ADAM_NO_MOMENTUM = {"lr": 0.002, "beta_1": 0.0, "beta_2": 0.95, "epsilon": 1e-5}
TINY = dict(n_movies=3, n_users=5)      # every id repeats in every batch, across its CTAs

TTCase = collections.namedtuple("TTCase", "over B n epochs seed adam")


def _tt(E, hidden, B, n, seed, adam=None, epochs=1, **vocab):
    return TTCase(dict(emb_dim=E, hidden=hidden, **vocab), B, n, epochs, seed, adam)


# the step's shared memory per case (restated by `step_smem_bytes` below) is in the comment
TT_MATRIX = [
    _tt(1, (1,), 65, 615, 0),                                    # <12, 16>   24.2 KiB
    _tt(12, (17, 9), 129, 1231, 1, ADAM),                        # <12, 32>   82.0 KiB
    _tt(13, (16, 16), 65, 300, 2, epochs=2),                     # <16, 16>   44.8 KiB, just under the opt-in
    _tt(16, (32, 32, 32), 129, 1231, 3, ADAM),                   # <16, 32>  125.3 KiB
    _tt(17, (1,), 65, 615, 4, ADAM_NO_MOMENTUM),                 # <32, 16>   36.7 KiB
    _tt(32, (17, 9), 65, 615, 5),                                # <32, 32>   97.0 KiB
    _tt(32, (9, 32, 17), 129, 600, 6, ADAM, epochs=2),           # <32, 32>  137.3 KiB: the opt-in grows
    _tt(33, (16, 16, 16), 65, 615, 7),                           # <64, 16>   92.9 KiB
    _tt(64, (32, 32, 32), 129, 1231, 8, ADAM),                   # <64, 32>  161.3 KiB, the largest step
    _tt(64, (32, 17), 200, 1877, 9, ADAM, **TINY),               # <64, 32>  121.0 KiB, below the size opted in
]


def _adam_id(adam):
    return "keras" if adam is None else "b1_0" if adam["beta_1"] == 0 else "adam"


def case_id(c):
    parts = ["E%d" % c.over["emb_dim"], "h" + "x".join(map(str, c.over["hidden"])), "B%d" % c.B, "n%d" % c.n]
    if c.epochs != 1:
        parts.append("ep%d" % c.epochs)
    if "n_movies" in c.over:
        parts.append("V%dx%d" % (c.over["n_movies"], c.over["n_users"]))
    return "-".join(parts + [_adam_id(c.adam), "s%d" % c.seed])


def case_spec(c):
    return default_spec("twotowers", **dict(dict(n_movies=N_MOVIES, n_users=N_USERS, final_dense=True), **c.over))


def steps(c):
    return c.epochs * -(-c.n // c.B)


def round_ep(E):
    """The trainer's padded embedding width (csrc/placement.h round_ep)."""
    return 12 if E <= 12 else 16 if E <= 16 else 32 if E <= 32 else 64


def instantiation(c):
    """(EP, HP) of the step a case runs, by srs_trainer_create's rule: HP = 16 if the widest hidden layer is at most
    16, else 32."""
    spec = case_spec(c)
    return round_ep(spec.emb_dim), 16 if max(spec.hidden) <= 16 else 32


def step_smem_bytes(c, n_layers=None):
    """csrc/twotowers_train.cu step_smem_bytes: place_ncf's two-tower blob (per tower a first kernel [EP][HP], each
    later kernel [HP][HP], a bias [HP] per layer; then dense_out's kernel and bias, 4 floats each) and, per row of the
    64-row CTA, both embedding rows [2EP], each tower's per-layer output and delta [HP], the Dot and dL/dz."""
    EP, HP = instantiation(c)
    L = len(c.over["hidden"]) if n_layers is None else n_layers
    blob = 2 * (EP * HP + HP + (L - 1) * (HP * HP + HP)) + 8
    return 4 * (blob + TILE_ROWS * (2 * EP + 4 * L * HP + 2))


def dispatched():
    """The (EP, HP) pairs of `SRS_TT_STEP_CASE` (the step's dispatch) and of `SRS_NCF_CASE` (ncf_kernel's), read from
    csrc/*.cu."""
    tt, ncf = set(), set()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        with open(path) as f:
            src = f.read()
        tt |= {(int(e), int(h)) for e, h in re.findall(r"SRS_TT_STEP_CASE\((\d+), (\d+)\)", src)}
        ncf |= {(int(e), int(h)) for e, h in re.findall(r"SRS_NCF_CASE\((\d+), (\d+)\)", src)}
    return tt, ncf


# ---- the inputs and the oracle's fits ------------------------------------------------------------------
def _per_case(fn):
    memo = {}

    @functools.wraps(fn)
    def once(case):
        key = case_id(case)
        if key not in memo:
            memo[key] = fn(case)
        return memo[key]
    return once


@functools.lru_cache(maxsize=None)
def trainset():
    z = np.load(os.path.join(GOLDEN, "neuralcf_trainset.npz"))
    return {k: z[k] for k in ("movieId", "userId", "label")}


@_per_case
def inputs(c):
    """(W0, rows, orders) of a case: the reference initialisers with test biases at the case's seed, the golden
    training rows with their ids taken modulo the case's vocabularies, one permutation per epoch."""
    spec = case_spec(c)
    ts = trainset()
    f = {k: np.ascontiguousarray(ts[k][:c.n]) for k in ("movieId", "userId", "label")}
    f["movieId"] = (f["movieId"] % spec.n_movies).astype(np.int32)
    f["userId"] = (f["userId"] % spec.n_users).astype(np.int32)
    return init_weights(spec, c.seed, for_test=True), f, ncf_train.epoch_orders(c.n, c.epochs, 11)


def oracle_fit(c, dtype, adam):
    W0, f, orders = inputs(c)
    return twotowers_train.fit(W0, f["movieId"], f["userId"], f["label"], orders, c.B, dtype, hp=adam)[0]


@_per_case
def oracle(c):
    """(W64, W32, tolerance per tensor): the case's fit at float64 and float32, and the GPU's allowance, 4x the
    float32 fit's distance from the float64 one plus one float32 ulp of the tensor's largest value."""
    W64, W32 = oracle_fit(c, np.float64, c.adam), oracle_fit(c, np.float32, c.adam)
    tol = {k: SPREAD_MULTIPLE * float(np.abs(W32[k] - W64[k]).max())
           + float(np.spacing(np.float32(np.abs(W64[k]).max()))) for k in W64}
    return W64, W32, tol


# ---- the oracle ----------------------------------------------------------------------------------------
def small_case(seed, B, hidden=(6, 5), E=3, Vm=7, Vu=9):
    spec = default_spec("twotowers", emb_dim=E, n_movies=Vm, n_users=Vu, hidden=hidden, final_dense=True)
    W = {k: v.astype(np.float64) for k, v in init_weights(spec, seed, for_test=True).items()}
    rng = np.random.default_rng(seed + 100)
    for k in W:                                               # larger scale, so relus switch on both sides
        W[k] = W[k] * 2.0 + (rng.normal(0, 0.3, W[k].shape) if k.endswith("bias") else 0)
    mid = rng.integers(0, Vm, B)
    uid = rng.integers(0, Vu, B)
    mid[: B // 2] = mid[0]                                    # repeated ids
    uid[B // 2:] = uid[-1]
    y = rng.integers(0, 2, B)
    return spec, W, mid, uid, y


@pytest.mark.parametrize("seed,B,hidden", [(0, 1, (6, 5)), (1, 5, (4,)), (2, 12, (6, 5)), (3, 33, (3, 4, 5))])
def test_backward_matches_central_differences(seed, B, hidden):
    _, W, mid, uid, y = small_case(seed, B, hidden)
    g, _, _ = twotowers_train.gradients(W, mid, uid, y, np.float64)
    assert g.keys() == W.keys()
    h = 1e-6
    for name, w in W.items():
        num = np.zeros_like(w)
        for i in np.ndindex(w.shape):
            old = w[i]
            w[i] = old + h
            lp = twotowers_train.batch_loss(W, mid, uid, y)
            w[i] = old - h
            lm = twotowers_train.batch_loss(W, mid, uid, y)
            w[i] = old
            num[i] = (lp - lm) / (2 * h)
        np.testing.assert_allclose(g[name], num, rtol=1e-5, atol=1e-8, err_msg=name)


def test_partial_last_batch_divides_by_its_own_size():
    _, W, mid, uid, y = small_case(4, 12)
    order = np.arange(12)[None, :]
    # 12 rows at batch 5: steps of 5, 5 and 2 rows; the third step's gradient is the mean over its 2 rows
    W5, _, _, _ = twotowers_train.fit(W, mid, uid, y, order, 5, np.float64, max_steps=2)
    g, _, _ = twotowers_train.gradients(W5, mid[10:], uid[10:], y[10:], np.float64)
    g2 = [twotowers_train.gradients(W5, mid[i:i + 1], uid[i:i + 1], y[i:i + 1], np.float64)[0] for i in (10, 11)]
    for k in g:
        np.testing.assert_allclose(g[k], (g2[0][k] + g2[1][k]) / 2, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_forward_is_the_serving_oracle(dtype):
    spec, W, mid, uid, _ = small_case(8, 40)
    W = {k: v.astype(np.float32) for k, v in W.items()}
    p, z, _ = twotowers_train.forward(W, mid, uid, dtype)
    po, zo = ctr_oracle.twotowers_forward(spec, W, {"movieId": mid, "userId": uid}, dtype)
    assert np.array_equal(p, po[:, 0]) and np.array_equal(z, zo[:, 0])


def test_adam_first_step_moves_each_parameter_by_lr_sign_g():
    _, W, mid, uid, y = small_case(5, 12)
    g, _, _ = twotowers_train.gradients(W, mid, uid, y, np.float64)
    W1 = {k: v.copy() for k, v in W.items()}
    twotowers_train.Adam(W1, np.float64).step(W1, g)
    for k in W:
        d = W1[k] - W[k]
        # t = 1: m = 0.1 g, v = 0.001 g^2, alpha = lr sqrt(0.001) / 0.1, so the step is
        # lr g / (|g| + epsilon / sqrt(0.001)): lr sign(g) once |g| >> 3.2e-6
        np.testing.assert_allclose(d, -0.001 * g[k] / (np.abs(g[k]) + 1e-7 / np.sqrt(0.001)), rtol=1e-9,
                                   atol=1e-18, err_msg=k)
        big = np.abs(g[k]) > 1e-3
        assert big.any(), k
        np.testing.assert_allclose(d[big], -0.001 * np.sign(g[k][big]), rtol=4e-3, err_msg=k)
        assert np.all(d[g[k] == 0] == 0), k


def test_float32_oracle_tracks_float64():
    _, W, mid, uid, y = small_case(7, 40)
    orders = ncf_train.epoch_orders(40, 2, 7)
    W64, h64, _, _ = twotowers_train.fit(W, mid, uid, y, orders, 12, np.float64)
    W32, h32, _, _ = twotowers_train.fit(W, mid, uid, y, orders, 12, np.float32)
    for k in W:
        assert np.abs(W32[k] - W64[k]).max() < 1e-5, k
    assert abs(h32[-1]["loss"] - h64[-1]["loss"]) < 1e-5


def test_golden_fixture():
    with open(os.path.join(GOLDEN, "twotowers_fit.json")) as f:
        fit = json.load(f)
    assert (fit["model"], fit["emb_dim"], fit["hidden"], fit["final_dense"]) == ("twotowers", 10, [10, 10], True)
    assert fit["rows"] == 88827 and fit["epochs"] == 5 and fit["batch_size"] == 12
    assert [r["seed"] for r in fit["runs"]] == fit["seeds"] == [0, 1, 2, 3]
    for r in fit["runs"]:
        assert r["iterations"] == 5 * 7403 and len(r["history"]) == 5
        for k, (lo, hi) in fit["band"].items():
            assert lo <= r["test"][k] <= hi
    assert fit["band"]["roc_auc"][0] > 0.6, "the oracle's runs learn"


# ---- the trainer ABI's and the Python surfaces' rejections that need no device --------------------------
def _lib_or_skip():
    from sparrowrecsys_b200 import _lib
    try:
        return _lib, _lib.load()
    except ImportError as e:
        pytest.skip(str(e))


def _create_any(spec, hp=None):
    _lib, lib = _lib_or_skip()
    from sparrowrecsys_b200.model import _spec_struct
    sp = _spec_struct(spec)
    out = C.c_void_p()
    rc = lib.srs_trainer_create_any(C.byref(sp), None, 0, 0, None if hp is None else C.byref(hp), C.byref(out))
    assert not out.value
    return _lib, lib, rc


@pytest.mark.parametrize("overrides,match", [
    (dict(final_dense=False), b"final Dense"), (dict(hidden=(33,)), b"1..32"), (dict(hidden=(10, 33)), b"1..32"),
    (dict(hidden=(10, 10, 10, 10)), b"1..3 hidden layers")])
def test_trainer_rejects_unsupported_two_tower_shapes(overrides, match):
    _lib, lib, rc = _create_any(default_spec("twotowers", **overrides))
    assert rc == _lib.SRS_ERR_INVALID and match in lib.srs_last_error()


@pytest.mark.parametrize("hp", [dict(lr=0.0), dict(beta_1=1.0), dict(beta_2=-0.1), dict(epsilon=0.0)])
def test_trainer_rejects_bad_adam_hyperparameters(hp):
    _lib, _ = _lib_or_skip()
    _lib, lib, rc = _create_any(default_spec("twotowers", hidden=(10, 10)),
                                _lib.SrsAdam(**dict(ncf_train.KERAS_ADAM, **hp)))
    assert rc == _lib.SRS_ERR_INVALID and b"Adam" in lib.srs_last_error()


def test_python_trainer_rejects_the_raw_dot_before_any_device_call():
    _lib_or_skip()
    from sparrowrecsys_b200.training import Trainer
    assert "twotowers" in Trainer.MODELS
    spec = default_spec("twotowers", final_dense=False)
    with pytest.raises(ValueError, match="final Dense"):
        Trainer(spec, init_weights(spec, 0, for_test=False))


def test_the_tfrecmodel_surface_still_does_not_fit_and_names_the_trainer():
    from tfrecmodel import twotowers
    with pytest.raises(NotImplementedError, match="NeuralCF") as e:
        twotowers.fit({"movieId": np.zeros(1, np.int32)})
    assert "training.Trainer" in str(e.value)


# ---- the matrix is complete, and its tolerances see the defects ----------------------------------------
def test_dispatch_lines_are_ncf_kernels_and_each_is_reached():
    """The step dispatches exactly `ncf_kernel`'s (EP, HP) pairs, and some TT_MATRIX case runs each of them: a new
    instantiation without a case fails here."""
    tt, ncf = dispatched()
    assert len(tt) == 8 and tt == ncf, (tt, ncf)
    reached = {instantiation(c) for c in TT_MATRIX}
    assert not tt - reached, "no TT_MATRIX case runs <EP, HP> = %s" % sorted(tt - reached)


def test_matrix_covers_edges_widths_depths_and_batches():
    Es = {c.over["emb_dim"] for c in TT_MATRIX}
    assert {1, 12, 13, 16, 17, 32, 33, 64} <= Es, sorted(Es)
    assert {1, 16, 17, 32} <= {h for c in TT_MATRIX for h in c.over["hidden"]}
    assert {len(c.over["hidden"]) for c in TT_MATRIX} == {1, 2, 3}
    assert {65, 129, 200} <= {c.B for c in TT_MATRIX}
    for c in TT_MATRIX:
        assert c.B > TILE_ROWS and c.B % TILE_ROWS != 0, (case_id(c), "the batch must straddle the row tile")
        assert c.n % c.B != 0, (case_id(c), "the last batch must be partial")
        assert 8 <= steps(c) <= 12, (case_id(c), steps(c))
    adams = [_adam_id(c.adam) for c in TT_MATRIX]
    assert "b1_0" in adams and "adam" in adams and 0.3 <= adams.count("keras") / len(adams) <= 0.7, adams
    assert any(c.epochs == 2 for c in TT_MATRIX)
    assert any(case_spec(c).n_movies <= 3 and case_spec(c).n_users <= 5 and c.B > 2 * TILE_ROWS for c in TT_MATRIX)
    assert len({case_id(c) for c in TT_MATRIX}) == len(TT_MATRIX)


def test_matrix_crosses_the_shared_memory_opt_in_and_grows_it():
    """Cases on both sides of 48 KiB, the largest instantiation at its three-layer size within an H100 CTA's limit,
    and an instantiation run at a shape followed (in the order the GPU tests run) by a larger one."""
    smem = [step_smem_bytes(c) for c in TT_MATRIX]
    assert any(s <= OPT_IN_BYTES for s in smem) and any(s > OPT_IN_BYTES for s in smem), smem
    assert max(step_smem_bytes(c, 3) for c in TT_MATRIX) <= SMEM_LIMIT
    grows = [(i, j) for i in range(len(TT_MATRIX)) for j in range(i + 1, len(TT_MATRIX))
             if instantiation(TT_MATRIX[i]) == instantiation(TT_MATRIX[j]) and OPT_IN_BYTES < smem[i] < smem[j]]
    assert grows, "no instantiation is opted in and then asked for more"


@pytest.mark.parametrize("case", TT_MATRIX, ids=case_id)
def test_float64_oracle_moves_every_tensor(case):
    """A unit dead on every row of every batch leaves its chain without a gradient, and then a GPU fit that lost
    that chain would pass; each case's rows and seed move every tensor by many tolerances."""
    W0 = inputs(case)[0]
    W64, _, tol = oracle(case)
    for k in W0:
        moved = float(np.abs(W64[k] - W0[k]).max())
        assert moved > DEFECT_MULTIPLE * tol[k], (k, moved, tol[k])


def _defects(case):
    """(name, gradients function, Adam) of the defects a step could have, each injected through the module global
    `gradients` that the oracle's `fit` calls."""
    intact = twotowers_train.gradients
    E, hidden = case.over["emb_dim"], case.over["hidden"]

    def edited(edit):
        def grads(W, *args):
            out = intact(W, *args)
            edit(out[0])
            return out
        return grads

    def column(g):
        for k in twotowers_train.TABLES:
            g[k][:, E - 1] = 0

    def unit(g):
        for side in ("item", "user"):
            for l, h in enumerate(hidden):
                g["%s_dense_%d/kernel" % (side, l)][:, h - 1] = 0
                g["%s_dense_%d/bias" % (side, l)][h - 1] = 0

    def last_row(W, mid, uid, y, dtype):
        out = intact(W, mid, uid, y, dtype)
        B = len(y)
        if B > 1:
            g = intact(W, mid[:-1], uid[:-1], y[:-1], dtype)[0]
            out = ({k: v * ((B - 1) / B) for k, v in g.items()},) + tuple(out[1:])
        return out

    yield "embedding column %d gets no gradient" % (E - 1), edited(column), case.adam
    yield "the last unit of each hidden layer gets no gradient", edited(unit), case.adam
    yield "the last row of each batch is left out", last_row, case.adam
    yield "the other Adam", intact, ADAM if case.adam is None else None


@pytest.mark.parametrize("case", TT_MATRIX, ids=case_id)
def test_tolerance_sees_each_defect(case):
    """Each defect moves some tensor of the float64 fit by more than 10x the parity tolerance of the GPU test."""
    W64, _, tol = oracle(case)
    intact = twotowers_train.gradients
    for name, grads, adam in _defects(case):
        twotowers_train.gradients = grads
        try:
            Wd = oracle_fit(case, np.float64, adam)
        finally:
            twotowers_train.gradients = intact
        far, k = max((float(np.abs(Wd[k] - W64[k]).max()) / tol[k], k) for k in tol)
        assert far > DEFECT_MULTIPLE, "%s moves %s by only %.3g tolerances" % (name, k, far)
