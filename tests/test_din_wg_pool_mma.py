"""din_wg_kernel pools the history on a warpgroup MMA: D = A^T Pb, A the gathered history tile read MN-major
(its 128-byte rows are positions) and Pb the gate weights split to bf16, row 0 w hi and row 1 w lo.  The pooled
vector is h_hi w_hi + h_lo w_hi + h_hi w_lo: w rounded to 16 significant bits and h_lo w_lo dropped, the trade
the activation unit already makes (DESIGN.md section 4.1).

* CPU: `oracle/tc_precision.py` pools in fp32 with an exact w.  Emulating the split-w pooling instead keeps the
  logit within tol / 3 of the float64 oracle (0.27 tol on the cfg 3-shaped case, whose amplified table puts the
  pooled vector's rounding on the logit; 0.15 tol at most on test_tensor_core_precision's DIN cases), while a
  kernel that lost w lo would move it by more than 10 x tol.
* GPU: a known-answer check of the MN-major `m64n8k16` wrapper (`srs_selftest_wgmma` with N = 8), and the
  kernel at cfg 3's shape and at T in {9, 50, 63, 65, 129} against the float64 oracle.
"""
import numpy as np
import pytest

from oracle import tc_precision as P
from test_tensor_core_precision import DIN_WG, _case, _features, _oracle, _spec, _weights, prob_tol

# cfg 3: E = 32, T = 50; the others cover one partial tile, a tile one short of full, a ring of two tiles with
# one position in the last, and three tiles; E = 17 and 24 pad to 32, E = 33 and 64 take the EP = 64 path
CASES = [
    _case("din", DIN_WG, 32, (128, 64), 129, T=50, logit_tol=0.0002),
    _case("din", DIN_WG, 32, (128, 64), 65, T=9, logit_tol=0.0003),
    _case("din", DIN_WG, 24, (128, 64), 65, sms=1, T=63, logit_tol=0.0005),
    _case("din", DIN_WG, 32, (128, 64), 65, T=65, logit_tol=0.0002),
    _case("din", DIN_WG, 17, (128, 64), 31, T=129, logit_tol=0.0005),
    _case("din", DIN_WG, 64, (128, 64), 65, T=50, logit_tol=0.0005),
    _case("din", DIN_WG, 33, (128, 64), 65, sms=1, T=65, logit_tol=0.0005),
]
CFG3 = CASES[0]


def _case_id(c):
    return "E%d-T%d-B%d-sms%d" % (c.E, c.T, c.B, c.sms)


def _split_w_pooling(monkeypatch, keep_w_lo=True):
    """Route the emulation's pooling (einsum 'bt,btk->bk' of the gate weights and the split tile h = hi + lo)
    through the kernel's arithmetic: h_hi w_hi + h_lo w_hi + h_hi w_lo, or without the w lo term.  Returns the
    list the pooling calls are counted in, so that a caller can tell the rerouting took effect."""
    einsum = np.einsum
    calls = []

    def pooled(subscripts, *ops, **kw):
        if subscripts != "bt,btk->bk":
            return einsum(subscripts, *ops, **kw)
        calls.append(subscripts)
        w, h = ops
        w_hi, w_lo = P.split(w)
        h_hi, h_lo = P.split(h)
        out = einsum(subscripts, w_hi, h_hi + h_lo)
        if keep_w_lo:
            out = out + einsum(subscripts, w_lo, h_hi)
        return out

    monkeypatch.setattr(np, "einsum", pooled)
    return calls


def _logit(c, W, f):
    return P.forward(_spec(c), W, f)[1]


@pytest.mark.parametrize("case", [CFG3, CASES[-1]], ids=_case_id)
def test_split_w_pooling_within_tolerance(case, monkeypatch):
    W, f = _weights(case), _features(case)
    _, zo = _oracle(case, W, f)
    with monkeypatch.context() as m:
        calls = _split_w_pooling(m)
        zs = _logit(case, W, f)
    assert calls, "the emulation's pooling no longer goes through the split-w arithmetic"
    intact = np.abs(zs - zo).max()
    assert intact <= case.logit_tol / 3, "split-w pooling off by %.3g" % intact


def test_lost_w_lo_is_seen():
    """On the cfg 3-shaped case, a kernel that pooled with w hi alone would miss the tolerance by 10x."""
    case = CFG3
    W, f = _weights(case), _features(case)
    _, zo = _oracle(case, W, f)
    mp = pytest.MonkeyPatch()
    try:
        calls = _split_w_pooling(mp, keep_w_lo=False)
        zd = _logit(case, W, f)
    finally:
        mp.undo()
    assert calls, "the emulation's pooling no longer goes through the split-w arithmetic"
    moved = np.abs(zd - zo).max()
    assert moved > 10 * case.logit_tol, "lost w lo moves the logit by %.3g x tol" % (moved / case.logit_tol)


def _bf16_trunc(x):
    return (x.astype(np.float32).view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("KB", [1, 2, 4])
def test_mn_major_m64n8_known_answer(KB):
    import torch
    from sparrowrecsys_b200 import _lib
    rng = np.random.default_rng(80 + KB)
    K = 64 * KB
    A = rng.standard_normal((128, K)).astype(np.float32)
    B = rng.standard_normal((8, K)).astype(np.float32)
    dA, dB = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    dD = torch.zeros(128, 8, dtype=torch.float32, device="cuda:0")
    _lib.check(_lib.load().srs_selftest_wgmma(dA.data_ptr(), dB.data_ptr(), dD.data_ptr(), 8, KB, 0, 0))
    ref = _bf16_trunc(A).astype(np.float64) @ _bf16_trunc(B).astype(np.float64).T
    err = np.abs(dD.cpu().numpy() - ref).max()
    assert err < 1e-4 * max(1.0, np.abs(ref).max()), "max err %g (KB=%d)" % (err, KB)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_kernel_matches_float64_oracle(case):
    from sparrowrecsys_b200.model import CTRModel
    spec, W, f = _spec(case), _weights(case), _features(case)
    with CTRModel(spec, W, device=0) as m:
        assert m.kernel_name == case.kernel
        if case.sms:
            m.set_sm_limit(case.sms)
        p, z = m.predict_with_logits(f)
        p2, z2 = m.predict_with_logits(f)
        m.status()
    assert np.array_equal(p, p2) and np.array_equal(z, z2)
    po, zo = _oracle(case, W, f)
    err_z, err_p = np.abs(z - zo).max(), np.abs(p - po).max()
    print("%s logit err %.3g (tol %.3g)" % (_case_id(case), err_z, case.logit_tol))
    assert err_z <= case.logit_tol, "logit err %g" % err_z
    assert err_p <= prob_tol(case), "prob err %g" % err_p
