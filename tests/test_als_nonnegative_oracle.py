"""Nonnegative ALS (Spark's NNLSSolver): the oracles (oracle/als_nnls.py, oracle/als_nnls_c.c) against each other bit
for bit, every half-step's solution against the optimality conditions of its own system and against
scipy.optimize.nnls, deliberate mutations of the rule, hand-built corner cases, and the ABI's device-free
rejections.  DESIGN.md section 4.21 gives the semantics and the tolerances."""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import cholesky, solve_triangular
from scipy.optimize import nnls as scipy_nnls

from oracle import als as A
from oracle import als_cext as X
from oracle import als_implicit as I
from oracle import als_nnls as N
from oracle import als_nnls_cext as XN
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import collab

from test_als_implicit_oracle import implicit_cases
from test_als_oracle import bits, fixture_ratings, hand_cases, same_fit, singular_case

# Optimality tolerances, relative to each system's scale |A|max |x|max + |b|max (DESIGN.md section 4.21).  Over the
# fixture's four half-steps at rank 10, explicit and implicit, the largest KKT violation measured is 6.5e-7 and the
# largest gap to scipy's optimum 1.7e-5 (relative to |x*|max): NNLS.solve stops at a step below 1e-7, not at the
# optimum.  Each tolerance is about 6 to 8 times its measured gap.
KKT_TOL = 5e-6
OPT_TOL = 1e-4


def nnls_cases():
    """name -> (user, movie, rating, reg_param): the corner cases of the nonnegative solve."""
    cases = {}
    for name, (u, m, r) in hand_cases().items():
        cases[name] = (u, m, r, 0.05)
    rng = np.random.default_rng(21)
    # user 977 rates only below zero: once the movies are >= 0 its atb is <= 0 and its factor exactly 0; movie 400
    # is rated 0 by everyone: atb = 0
    u = rng.integers(1, 60, 900)
    m = rng.integers(1, 40, 900)
    r = rng.integers(1, 11, 900) / 2.0
    u = np.r_[u, 977, 977, 977, 5, 6, 7]
    m = np.r_[m, 3, 5, 8, 400, 400, 400]
    r = np.r_[r, -1.0, -2.5, -0.5, 0.0, 0.0, 0.0]
    cases["non_positive_rhs"] = (u, m, r, 0.05)
    su, sm, sr = singular_case()                           # user 9's system is all zero at reg 0
    cases["all_zero_system"] = (su, sm, sr, 0.0)
    rng = np.random.default_rng(0)                         # at rank 64 some movie's NNLS runs to iterMax
    cases["ill_conditioned"] = (rng.integers(0, 80, 2500), rng.integers(0, 60, 2500),
                                rng.integers(1, 11, 2500) / 2.0, 1e-9)
    return cases


def chunk_edge_case():
    """Movies with 31, 32, 33, 64 and 65 ratings (and users with as many), around the 32-rating staging chunk."""
    rng = np.random.default_rng(8)
    u, m = [], []
    for movie, n in zip((1, 2, 3, 4, 5), (31, 32, 33, 64, 65)):
        u += list(range(100, 100 + n))
        m += [movie] * n
    for user, n in zip((1, 2, 3, 4, 5), (31, 32, 33, 64, 65)):
        u += [user] * n
        m += list(range(200, 200 + n))
    u, m = np.array(u), np.array(m)
    return u, m, rng.integers(1, 11, len(u)) / 2.0


def _dense_system(lay, srcF, k, reg, alpha=None):
    """The system of one half-step in plain numpy, in any order: (sum y y^T + lambda n I, sum r y) explicit, or
    (Y^T Y + sum c1 y y^T + lambda n+ I, sum_{r>0} (1 + c1) y) implicit."""
    off, src, r = lay
    Y = srcF.astype(np.float64)
    base = Y.T @ Y if alpha is not None else np.zeros((k, k))
    out_a, out_b = [], []
    for e in range(len(off) - 1):
        ys, rv = Y[src[off[e]:off[e + 1]]], r[off[e]:off[e + 1]].astype(np.float64)
        if alpha is None:
            a, b, n = ys.T @ ys, ys.T @ rv, len(rv)
        else:
            c1 = alpha * np.abs(rv)
            a, b, n = base + (ys * c1[:, None]).T @ ys, ys.T @ np.where(rv > 0, 1 + c1, 0.0), int(np.sum(rv > 0))
        out_a.append(a + reg * n * np.eye(k))
        out_b.append(b)
    return np.array(out_a), np.array(out_b)


def _half_steps(u, m, r, k, reg, alpha, iters, seed=0):
    """Yields (layout, source factors, source ids, system A, b, x double) for each half-step of the C oracle's fit."""
    uids, mids, by_movie, by_user = A.layouts(u, m, r)
    U = X.init_user_factors(uids, k, seed)
    M = None
    for h in range(2 * iters):
        lay, src, ids = (by_movie, U, uids) if h % 2 == 0 else (by_user, M, mids)
        if alpha is None:
            Am, B = A.normal_equations(lay, src, k, reg)
        else:
            Am, B = I.normal_equations(lay, src, ids, k, reg, alpha)
        Am = np.triu(Am) + np.transpose(np.triu(Am, 1), (0, 2, 1))
        x, _ = N.nnls(Am, B)
        out, _ = XN.solve_half(lay, src, ids, k, reg, alpha)
        assert np.array_equal(bits(out), bits(x.astype(np.float32)))
        Ad, Bd = _dense_system(lay, src, k, reg, alpha)
        yield lay, src, ids, Ad, Bd, x
        if h % 2 == 0:
            M = out
        else:
            U = out


def kkt_violation(Ad, Bd, x):
    """Per entity, the largest violation of x >= 0, g_i >= 0 where x_i = 0 and g_i = 0 where x_i > 0 (g = A x - b),
    relative to the system's scale."""
    g = np.einsum("eij,ej->ei", Ad, x) - Bd
    scale = np.abs(Ad).max(axis=(1, 2)) * np.abs(x).max(axis=1) + np.abs(Bd).max(axis=1)
    scale = np.where(scale > 0, scale, 1.0)
    v = np.where(x > 0, np.abs(g), np.maximum(-g, 0.0))
    v = np.maximum(v, np.maximum(-x, 0.0))
    return v.max(axis=1) / scale


def optimum_gap(Ad, Bd, x):
    """Per entity, |x - x*|max / |x*|max against scipy.optimize.nnls on the Cholesky-transformed system: with
    A = L L^T, min 1/2 x^T A x - b^T x over x >= 0 is min |L^T x - L^-1 b| over x >= 0."""
    gaps = []
    for a, b, xe in zip(Ad, Bd, x):
        L = cholesky(a, lower=True)
        xs, _ = scipy_nnls(L.T, solve_triangular(L, b, lower=True), maxiter=50 * len(b))
        gaps.append(np.abs(xe - xs).max() / max(np.abs(xs).max(), 1e-300) if np.any(xs) else np.abs(xe).max())
    return np.array(gaps)


# ---- numpy and C oracles ----------------------------------------------------------------------------------------
MODES = [None, 0.0, 1.0, 40.0]                              # explicit, then implicit at each alpha


def _kw(mode):
    return {} if mode is None else dict(implicit_prefs=True, alpha=mode)


@pytest.mark.parametrize("rank", [1, 10, 33, 64])
@pytest.mark.parametrize("max_iter", [1, 2])
@pytest.mark.parametrize("mode", MODES, ids=["explicit", "alpha0", "alpha1", "alpha40"])
def test_numpy_and_c_oracles_bit_equal_on_hand_built_cases(rank, max_iter, mode):
    cases = [(u, m, r, 0.05) for u, m, r in implicit_cases().values()] if mode is not None else []
    cases += [c for name, c in nnls_cases().items() if name != "ill_conditioned"]
    for u, m, r, reg in cases:
        kw = dict(rank=rank, max_iter=max_iter, reg_param=reg, seed=rank, **_kw(mode))
        same_fit(N.fit(u, m, r, **kw), XN.fit(u, m, r, **kw))


@pytest.mark.parametrize("max_iter", [1, 2])
@pytest.mark.parametrize("mode", [None, 1.0], ids=["explicit", "implicit"])
def test_numpy_and_c_oracles_bit_equal_on_the_fixture(max_iter, mode):
    r = fixture_ratings()
    kw = dict(rank=10, max_iter=max_iter, reg_param=0.01, seed=4, **_kw(mode))
    same_fit(N.fit(r["userId"], r["movieId"], r["rating"], **kw), XN.fit(r["userId"], r["movieId"], r["rating"], **kw))


def test_the_ill_conditioned_case_reaches_iter_max_and_both_oracles_agree():
    u, m, r, reg = nnls_cases()["ill_conditioned"]
    uids, mids, by_movie, _ = A.layouts(u, m, r)
    U = X.init_user_factors(uids, 64, 0)
    it = np.zeros(len(mids), np.int32)
    out, _ = XN.solve_half(by_movie, U, uids, 64, reg, None, it)
    assert (it == N.iter_max(64)).any() and (it < N.iter_max(64)).any()
    Am, B = A.normal_equations(by_movie, U, 64, reg)
    x, its = N.nnls(np.triu(Am) + np.transpose(np.triu(Am, 1), (0, 2, 1)), B)
    assert np.array_equal(its, it) and np.array_equal(bits(out), bits(x.astype(np.float32)))
    same_fit(N.fit(u, m, r, rank=64, max_iter=1, reg_param=reg), XN.fit(u, m, r, rank=64, max_iter=1, reg_param=reg))


# ---- optimality -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [None, 1.0], ids=["explicit", "implicit"])
def test_every_half_step_on_the_fixture_is_optimal(mode):
    r = fixture_ratings()
    for _, _, _, Ad, Bd, x in _half_steps(r["userId"], r["movieId"], r["rating"], 10, 0.01, mode, 2):
        assert np.all(x >= 0)
        assert kkt_violation(Ad, Bd, x).max() <= KKT_TOL
        assert optimum_gap(Ad, Bd, x).max() <= OPT_TOL


@pytest.mark.parametrize("name", ["one_rating_user", "duplicate_pairs", "non_positive_rhs"])
@pytest.mark.parametrize("rank", [4, 33])
def test_every_half_step_on_hand_built_cases_is_optimal(name, rank):
    u, m, r, reg = nnls_cases()[name]
    for mode in (None, 40.0):
        for _, _, _, Ad, Bd, x in _half_steps(u, m, r, rank, reg, mode, 2, seed=3):
            assert np.all(x >= 0)
            assert kkt_violation(Ad, Bd, x).max() <= KKT_TOL
            assert optimum_gap(Ad, Bd, x).max() <= OPT_TOL


# ---- mutants ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mutant", ["no_projection", "always_cg", "no_clip", "parallel_clip", "no_lambda"])
def test_each_mutation_of_the_rule_is_caught(mutant):
    """Each mutant differs from the C oracle in the bits, and fails the optimality check or the sign of x, on the
    fixture's first two half-steps."""
    r = fixture_ratings()
    reg = 0.01
    caught_bits = caught_opt = False
    for lay, src, ids, Ad, Bd, _ in _half_steps(r["userId"], r["movieId"], r["rating"], 10, reg, None, 1):
        want, _ = XN.solve_half(lay, src, ids, 10, reg)
        got, _ = N.solve_half(lay, src, ids, 10, reg, mutant=mutant)
        caught_bits |= not np.array_equal(bits(got), bits(want))
        with np.errstate(all="ignore"):
            x = got.astype(np.float64)
            caught_opt |= bool(np.any(~(x >= 0)) or np.any(~(kkt_violation(Ad, Bd, x) <= KKT_TOL)))
    assert caught_bits, mutant
    if mutant in ("no_clip", "no_lambda"):                  # these leave the orthant or solve another system
        assert caught_opt, mutant


# ---- hand-built cases -------------------------------------------------------------------------------------------
def test_a_non_positive_right_hand_side_gives_exactly_zero():
    rng = np.random.default_rng(4)
    Y = rng.normal(size=(30, 6))
    a = Y.T @ Y + 0.1 * np.eye(6)
    b = -np.abs(rng.normal(size=6))
    b[2] = 0.0
    x, it = N.nnls(a[None], b[None])
    assert np.all(x == 0) and not np.signbit(x).any() and it[0] == 0
    u, m, r, reg = nnls_cases()["non_positive_rhs"]
    for fit in (N.fit, XN.fit):
        uids, U, mids, M = fit(u, m, r, rank=5, max_iter=2, reg_param=reg, seed=1)
        assert np.all(U[np.searchsorted(uids, 977)] == 0)   # atb <= 0 once the movies are >= 0
        assert np.all(M[np.searchsorted(mids, 400)] == 0)   # atb = 0


def test_a_positive_unconstrained_solution_is_the_cholesky_answer():
    rng = np.random.default_rng(5)
    for k in (1, 4, 10, 33):
        Y = rng.normal(size=(3 * k + 5, k))
        a = Y.T @ Y + 0.05 * np.eye(k)
        want = rng.uniform(0.5, 2.0, k)
        b = a @ want
        x, it = N.nnls(a[None], b[None])
        ref = np.linalg.solve(a, b)
        assert np.all(ref > 0)
        assert np.abs(x[0] - ref).max() / np.abs(ref).max() <= OPT_TOL, k
    r = fixture_ratings()                                  # and in a fit: every strictly positive Cholesky solution
    for _, src, _, Ad, Bd, x in _half_steps(r["userId"], r["movieId"], r["rating"], 3, 0.01, None, 1):
        ref = np.linalg.solve(Ad, Bd[:, :, None])[:, :, 0]
        pos = np.all(ref > 0, axis=1)
        assert pos.sum() > 10
        rel = np.abs(x[pos] - ref[pos]).max(axis=1) / np.abs(ref[pos]).max(axis=1)
        assert rel.max() <= OPT_TOL


def test_regparam_zero_with_an_all_zero_system_is_not_an_error():
    x, it = N.nnls(np.zeros((1, 3, 3)), np.zeros((1, 3)))
    assert np.all(x == 0) and it[0] == 0
    u, m, r, reg = nnls_cases()["all_zero_system"]
    with pytest.raises(A.SingularError):
        X.fit(u, m, r, rank=2, max_iter=1, reg_param=reg)
    for fit in (N.fit, XN.fit):
        uids, U, _, _ = fit(u, m, r, rank=2, max_iter=1, reg_param=reg)
        assert np.all(U[np.searchsorted(uids, 9)] == 0)


def test_the_chunk_edge_case_has_its_counts():
    u, m, _ = chunk_edge_case()
    for side, ids in ((m, (1, 2, 3, 4, 5)), (u, (1, 2, 3, 4, 5))):
        assert [int(np.sum(side == i)) for i in ids] == [31, 32, 33, 64, 65]


# ---- Python surface without a device ----------------------------------------------------------------------------
def test_param_maps_take_nonnegative_and_still_reject_alpha():
    maps = collab.param_maps([("nonnegative", [False, True]), ("reg_param", [0.01, 0.1])])
    assert maps == [{"nonnegative": False, "reg_param": 0.01}, {"nonnegative": True, "reg_param": 0.01},
                    {"nonnegative": False, "reg_param": 0.1}, {"nonnegative": True, "reg_param": 0.1}]
    assert collab.param_maps([("reg_param", [0.01, 0.1])]) == [{"reg_param": 0.01}, {"reg_param": 0.1}]
    with pytest.raises(ValueError):
        collab.param_maps([("alpha", [1.0])])


def test_command_usage_errors_exit_2():
    assert collab.main(["r.csv", "--nonnegative", "--implicit", "--cv"]) == 2
    assert collab.main(["r.csv", "--nonnegative", "--alpha", "2"]) == 2
    assert collab.main(["--nonnegative"]) == 2


# ---- the ABI's device-free rejections ---------------------------------------------------------------------------
def _raw_nonneg(u, m, r, rank=10, max_iter=5, reg=0.01, implicit=0, alpha=1.0, cap=8):
    lib = _lib.load()
    u, m = np.ascontiguousarray(u, np.int32), np.ascontiguousarray(m, np.int32)
    r = np.ascontiguousarray(r, np.float32)
    p = _lib.SrsAlsParams(rank, max_iter, reg, 0)
    ui, mi = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    uf, mf = np.zeros((cap, 64), np.float32), np.zeros((cap, 64), np.float32)
    nu, nm = C.c_int32(-1), C.c_int32(-1)
    rc = lib.srs_als_fit_nonnegative_host(u.ctypes.data, m.ctypes.data, r.ctypes.data, len(u), C.byref(p), 0, cap,
                                          cap, ui.ctypes.data, uf.ctypes.data, C.byref(nu), mi.ctypes.data,
                                          mf.ctypes.data, C.byref(nm), implicit, alpha)
    return rc, nu.value, nm.value, lib.srs_last_error().decode()


def test_nonnegative_fit_rejects_bad_inputs_before_any_device_call():
    u, m, r = [1, 2], [3, 4], [4.0, 5.0]
    INV = _lib.SRS_ERR_INVALID
    for kw, word in ((dict(implicit=2), "implicit_prefs"), (dict(implicit=-1), "implicit_prefs"),
                     (dict(implicit=1, alpha=-0.5), "alpha"), (dict(implicit=1, alpha=float("nan")), "alpha"),
                     (dict(rank=0), "rank"), (dict(rank=65), "rank"), (dict(max_iter=0), "max_iter"),
                     (dict(reg=-1.0), "reg_param"), (dict(reg=float("inf")), "reg_param")):
        rc, nu, nm, msg = _raw_nonneg(u, m, r, **kw)
        assert (rc, nu, nm) == (INV, 0, 0) and word in msg, (kw, msg)
    rc, _, _, msg = _raw_nonneg(u, m, [4.0, float("nan")])
    assert rc == INV and "not finite" in msg
    assert _raw_nonneg([1, -2], m, r)[0] == INV
    assert _raw_nonneg([], [], [])[0] == INV


def _raw_folds(nonneg, models=None, fold=(0, 1), n_folds=2):
    lib = _lib.load()
    u, m = np.array([1, 2], np.int32), np.array([3, 4], np.int32)
    r = np.array([4.0, 5.0], np.float32)
    fold = np.ascontiguousarray(fold, np.int32)
    models = models or [(4, 1, 0.01, 0), (4, 1, 0.01, 1)]
    specs = (_lib.SrsAlsModel * len(models))(*[_lib.SrsAlsModel(*x) for x in models])
    cap = 4
    ui, mi = np.zeros((len(models), cap), np.int32), np.zeros((len(models), cap), np.int32)
    uf, mf = np.zeros(cap * 64 * len(models), np.float32), np.zeros(cap * 64 * len(models), np.float32)
    nu, nm = np.full(len(models), -1, np.int32), np.full(len(models), -1, np.int32)
    flags = None if nonneg is None else np.ascontiguousarray(nonneg, np.int32).ctypes.data
    rc = lib.srs_als_fit_folds_nonnegative_host(u.ctypes.data, m.ctypes.data, r.ctypes.data, fold.ctypes.data, 2,
                                                n_folds, specs, len(models), 0, 0, cap, cap, ui.ctypes.data,
                                                uf.ctypes.data, nu.ctypes.data, mi.ctypes.data, mf.ctypes.data,
                                                nm.ctypes.data, flags)
    return rc, nu, nm, lib.srs_last_error().decode()


def test_batched_nonnegative_fit_rejects_bad_inputs_before_any_device_call():
    INV = _lib.SRS_ERR_INVALID
    for flags, word in (([0, 2], "nonnegative"), ([-1, 1], "nonnegative"), (None, "nonnegative")):
        rc, nu, nm, msg = _raw_folds(flags)
        assert rc == INV and word in msg and np.all(nu == 0) and np.all(nm == 0), (flags, msg)
    rc, _, _, msg = _raw_folds([1, 1], models=[(0, 1, 0.01, 0), (4, 1, 0.01, 1)])
    assert rc == INV and "model 0" in msg and "rank" in msg
    rc, _, _, msg = _raw_folds([1, 0], models=[(4, 1, 0.01, 3), (4, 1, 0.01, 1)])
    assert rc == INV and "exclude_fold" in msg
    rc, _, _, msg = _raw_folds([1, 1], fold=(0, 2))
    assert rc == INV and "fold" in msg
