"""`model.fit` at every step-kernel instantiation, hidden depth and padding edge against the float64 training oracle.

NeuralCF's step is `ncf_train_step_kernel<EP, HP>` (EP in {12, 16, 32, 64}, HP in {16, 32}; csrc/ncf_train.cu) over
1 to 3 hidden layers; the trainer (csrc/trainer.cu) opts it into its three-layer dynamic shared memory at create,
which is above 48 KiB for some instantiations and covers every smaller shape.  DeepFM's is `deepfm_train_step_kernel<EP>`
(csrc/deepfm_train.cu), with the serving `deepfm_kernel<EP>` for validation and `Trainer.evaluate`.  The trainer places
its weights through the serving builders' placement (csrc/placement.h) and gathers its exports back through it, and
its step kernels restate the layout's offsets.  The defects such code invites - a padded column read as data, the last real column or unit dropped, the wrong
template, a tail tile mishandled - compound over a fit's steps.  `FIT_MATRIX` names one case per (model,
instantiation, width regime): the smallest E of a bucket, a partial pad and the exact bucket width, hidden width 1
and each model's limit, batches one row past the step's row tile or its double (64 rows for NeuralCF, 32 for DeepFM),
about ten steps with the last batch partial, Keras's Adam and custom Adam, and per model one tiny vocabulary whose
ids repeat across the CTAs of every batch (the row-order dedupe of `table_grad_kernel`).

* GPU, per case: the trainer exports its initial weights bit for bit; the fit matches the float64 oracle within 4x
  the float32 oracle's own distance from it (plus one ulp); the step's forward is the serving forward, number for
  number; after the fit, the trainer's evaluate is that of a serving model rebuilt (with zero padding) from its
  exported weights; a second fit gives the same bits.
* CPU: `FIT_MATRIX` reaches every instantiation the launchers dispatch, 1, 2 and 3 hidden layers, width 1 and each
  model's limit, both sides of the shared-memory opt-in and its growth; each case's tolerance sees a dropped
  embedding column, a dropped hidden unit, a dropped batch row and the other Adam; and the float64 oracle moves
  every tensor of every case, so that no dead unit leaves a chain untested.
"""
import collections
import functools
import glob
import os
import re

import numpy as np
import pytest

from oracle import deepfm_train, ncf_train
from sparrowrecsys_b200.spec import default_spec
from sparrowrecsys_b200.weights import init_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc")
N_MOVIES, N_USERS = 1000, 1200          # the kernel matrix's small vocabularies; the golden ids are taken modulo them
SPREAD_MULTIPLE = 4.0                   # GPU-to-float64 distance allowed, in units of the float32-to-float64 distance
DEFECT_MULTIPLE = 10.0                  # a defect must move some tensor by this many tolerances
OPT_IN_BYTES = 48 * 1024                # dynamic shared memory a kernel gets without cudaFuncSetAttribute
TILE_ROWS = {"neuralcf": 64, "deepfm": 32}
MAX_HIDDEN = {"neuralcf": 32, "deepfm": 64}
CUDACORE = {"deepfm_impl": "cudacore"}  # the serving kernel whose forward the DeepFM step shares
ADAM = {"lr": 0.003, "beta_1": 0.8, "beta_2": 0.99, "epsilon": 1e-6}
ADAM_NO_MOMENTUM = {"lr": 0.002, "beta_1": 0.0, "beta_2": 0.95, "epsilon": 1e-5}

FitCase = collections.namedtuple("FitCase", "model over B n epochs seed adam")


def _ncf(E, hidden, B, n, seed, adam=None, epochs=1, **vocab):
    return FitCase("neuralcf", dict(emb_dim=E, hidden=hidden, **vocab), B, n, epochs, seed, adam)


def _fm(E, hidden, B, n, seed, adam=None, epochs=1, **vocab):
    return FitCase("deepfm", dict(emb_dim=E, hidden=hidden, **vocab), B, n, epochs, seed, adam)


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
]


def _adam_id(adam):
    return "keras" if adam is None else "b1_0" if adam["beta_1"] == 0 else "adam"


def _case_id(c):
    parts = [c.model, "E%d" % c.over["emb_dim"], "h" + "x".join(map(str, c.over["hidden"])), "B%d" % c.B,
             "n%d" % c.n]
    if c.epochs != 1:
        parts.append("ep%d" % c.epochs)
    if "n_movies" in c.over:
        parts.append("V%dx%d" % (c.over["n_movies"], c.over["n_users"]))
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
    HP = 16 if its widest hidden layer is at most 16, else 32; DeepFM pads every hidden layer to 64."""
    spec = _spec(c)
    EP = round_ep(spec.emb_dim)
    if c.model == "neuralcf":
        return {("ncf_train_step_kernel", EP, 16 if max(spec.hidden) <= 16 else 32)}
    return {("deepfm_train_step_kernel", EP), ("deepfm_kernel", EP)}


def dispatched_instantiations():
    """Every instantiation the trainer's launchers in csrc/*.cu can dispatch, read from their dispatch lines: the step
    kernels' cases, and the cases of `launch_deepfm`'s switch (the trainer's DeepFM forward)."""
    found = set()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        with open(path) as f:
            src = f.read()
        for ep, hp in re.findall(r"SRS_TRAIN_CASE\((\d+), (\d+)\)", src):
            found.add(("ncf_train_step_kernel", int(ep), int(hp)))
        for ep in re.findall(r"SRS_DEEPFM_TRAIN_CASE\((\d+)\)", src):
            found.add(("deepfm_train_step_kernel", int(ep)))
        launcher = re.search(r"cudaError_t launch_deepfm\(const DeepFmParams& p.*?\n}", src, re.S)
        if launcher:
            for ep in re.findall(r"case (\d+): return launch_deepfm_t<(?:\d+)>", launcher.group(0)):
                found.add(("deepfm_kernel", int(ep)))
    return found


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


@_per_case
def _inputs(c):
    """(W0, rows, orders) of a case: the reference initialisers with test biases at the case's seed; the golden
    training rows with their ids taken modulo the case's vocabularies; one permutation per epoch."""
    spec = _spec(c)
    W0 = init_weights(spec, c.seed, for_test=True)
    ts = _trainset(c.model)
    if c.model == "neuralcf":
        f = {k: np.ascontiguousarray(ts[k][:c.n]) for k in ("movieId", "userId", "label")}
    else:
        f = _fm_rows(ts, c.n)
    f["movieId"] = (f["movieId"] % spec.n_movies).astype(np.int32)
    f["userId"] = (f["userId"] % spec.n_users).astype(np.int32)
    return W0, f, ncf_train.epoch_orders(c.n, c.epochs, 11)


def _oracle_fit(c, dtype, adam):
    W0, f, orders = _inputs(c)
    if c.model == "neuralcf":
        return ncf_train.fit(W0, f["movieId"], f["userId"], f["label"], orders, c.B, dtype, hp=adam)[0]
    return deepfm_train.fit(W0, deepfm_train.Rows.from_features(f), f["label"], orders, c.B, dtype, hp=adam)[0]


@_per_case
def _oracle(c):
    """(W64, W32, tolerance per tensor): the case's fit at float64 and float32, and the GPU's allowance, 4x the
    float32 fit's distance from the float64 one plus one float32 ulp of the tensor's largest value (no float32 result
    is nearer than that)."""
    W64, W32 = _oracle_fit(c, np.float64, c.adam), _oracle_fit(c, np.float32, c.adam)
    tol = {k: SPREAD_MULTIPLE * float(np.abs(W32[k] - W64[k]).max())
           + float(np.spacing(np.float32(np.abs(W64[k]).max()))) for k in W64}
    return W64, W32, tol


def _distance(Wa, Wb, tol):
    """(the largest distance in tolerances over the tensors, its tensor)."""
    return max((float(np.abs(Wa[k] - Wb[k]).max()) / tol[k], k) for k in tol)


# ---- CPU: the matrix is complete, and its tolerances see the defects -------------------------------------
def test_matrix_reaches_every_step_and_forward_instantiation():
    """Every step-kernel instantiation the trainer dispatches, and every `deepfm_kernel` instantiation (the trainer's
    DeepFM forward for validation and evaluate), is run by some FIT_MATRIX case."""
    dispatched = dispatched_instantiations()
    assert {d[0] for d in dispatched} == {"ncf_train_step_kernel", "deepfm_train_step_kernel",
                                          "deepfm_kernel"}, dispatched
    reached = set().union(*(instantiations(c) for c in FIT_MATRIX))
    missing = sorted(dispatched - reached)
    assert not missing, "no FIT_MATRIX case runs %s" % ", ".join("%s<%s>" % (d[0], ", ".join(map(str, d[1:])))
                                                                 for d in missing)


def test_matrix_covers_depths_widths_and_batches():
    for model in TILE_ROWS:
        cases = [c for c in FIT_MATRIX if c.model == model]
        widths = {h for c in cases for h in c.over["hidden"]}
        assert {1, MAX_HIDDEN[model]} <= widths, (model, widths)
        assert any(_spec(c).n_movies <= 3 and _spec(c).n_users <= 5 and c.B > 2 * TILE_ROWS[model] for c in cases), \
            "%s: no case whose ids repeat across the CTAs of a batch" % model
        for c in cases:
            tile = TILE_ROWS[model]
            assert c.B > tile and c.B % tile != 0, (_case_id(c), "the batch must straddle the row tile")
            assert c.n % c.B != 0, (_case_id(c), "the last batch must be partial")
            assert 8 <= _steps(c) <= 12, (_case_id(c), _steps(c))
    assert {len(c.over["hidden"]) for c in FIT_MATRIX if c.model == "neuralcf"} == {1, 2, 3}
    adams = [_adam_id(c.adam) for c in FIT_MATRIX]
    assert "b1_0" in adams and 0.3 <= adams.count("keras") / len(adams) <= 0.7, adams


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


@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_float64_oracle_moves_every_tensor(case):
    """A unit that is dead on every row of every batch leaves its chain without a gradient, and then a GPU fit that
    lost that chain would pass; each case's seed is chosen so that every tensor moves by many tolerances."""
    W0 = _inputs(case)[0]
    W64, _, tol = _oracle(case)
    for k in W0:
        moved = float(np.abs(W64[k] - W0[k]).max())
        assert moved > DEFECT_MULTIPLE * tol[k], (k, moved, tol[k])


def _defects(case):
    """(name, gradients function, Adam) of the defects a trainer could have, each injected through the module
    global `gradients` that the oracle's `fit` calls."""
    mod = ncf_train if case.model == "neuralcf" else deepfm_train
    intact = mod.gradients
    E, hidden = case.over["emb_dim"], case.over["hidden"]
    layers = ["dense_%d" % l for l in range(len(hidden))] if case.model == "neuralcf" else ["dense", "dense_1"]

    def column(*args):
        g, p, z = intact(*args)
        for k in g:
            if k.endswith("_embedding"):
                g[k][:, E - 1] = 0
        return g, p, z

    def unit(*args):
        g, p, z = intact(*args)
        for layer, h in zip(layers, hidden):
            g[layer + "/kernel"][:, h - 1] = 0
            g[layer + "/bias"].reshape(-1)[h - 1] = 0
        return g, p, z

    def last_row(W, *args):
        # NeuralCF: (mid, uid, y, dtype); DeepFM: (rows, y, dtype)
        *cols, dtype = args
        B = len(cols[0] if case.model == "neuralcf" else cols[0].mid)
        g, p, z = intact(W, *cols, dtype)
        if B > 1:
            if case.model == "neuralcf":
                head = [a[:-1] for a in cols]
            else:
                head = [cols[0].take(np.arange(B - 1)), cols[1][:-1]]
            g = {k: v * ((B - 1) / B) for k, v in intact(W, *head, dtype)[0].items()}
        return g, p, z

    yield "embedding column %d gets no gradient" % (E - 1), column, case.adam
    yield "the last unit of each hidden layer gets no gradient", unit, case.adam
    yield "the last row of each batch is left out", last_row, case.adam
    yield "the other Adam", intact, ADAM if case.adam is None else None


@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_tolerance_sees_each_defect(case):
    """Each defect moves some tensor of the float64 fit by more than 10x the parity tolerance of the GPU test."""
    mod = ncf_train if case.model == "neuralcf" else deepfm_train
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
    m = CTRModel(_spec(case), W, options=CUDACORE if case.model == "deepfm" else None)
    assert m.kernel_name == ("ncf_kernel<neural_cf_model_1>" if case.model == "neuralcf" else "deepfm_kernel")
    return m


def _same_result(r, s):
    assert (r.rows, r.positives, r.correct) == (s.rows, s.positives, s.correct)
    assert (r.loss, r.accuracy, r.roc_auc, r.pr_auc) == (s.loss, s.accuracy, s.roc_auc, s.pr_auc)


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
    """Every tensor within 4x the float32 oracle's spread (plus one ulp) of the float64 fit.  The test runs the cases
    in FIT_MATRIX's order in one process, so NeuralCF's <32, 32> opts in at 60.6 KiB and then grows to 80.8 KiB."""
    W0, f, orders = _inputs(case)
    W64, W32, tol = _oracle(case)
    with _trainer(case, W0) as tr:
        tr.fit(f, epochs=case.epochs, batch_size=case.B, order=orders)
        assert tr.iterations == _steps(case)
        Wg = tr.weights()
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
    model's evaluate of the same rows in one batch, number for number."""
    W0, f, _ = _inputs(case)
    with _trainer(case, W0) as tr:
        h = tr.fit(f, epochs=1, batch_size=case.n, order=[np.arange(case.n)])
    with _serving(case, W0) as m:
        loss, acc, roc, pr = m.evaluate(f, batch_size=case.n)
    assert (h["loss"][0], h["accuracy"][0], h["auc"][0], h["auc_1"][0]) == (loss, acc, roc, pr)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FIT_MATRIX, ids=_case_id)
def test_padding_stays_zero(case):
    """After the fit, the trainer's evaluate (its own padded arrays, through the NcfParams / DeepFmParams it keeps over
    them) is the evaluate of a serving model built from the exported weights, whose padding is zero by construction."""
    W0, f, orders = _inputs(case)
    with _trainer(case, W0) as tr:
        tr.fit(f, epochs=case.epochs, batch_size=case.B, order=orders)
        got = tr.evaluate_result(f)
        W = tr.weights()
    with _serving(case, W) as m:
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
