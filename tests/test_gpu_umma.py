"""Known-answer test of the tensor-core MMA building blocks (csrc/wgmma.cuh: warpgroup MMAs) on the H100."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _bf16_trunc(x):
    return (x.astype(np.float32).view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


@pytest.mark.parametrize("a_in_regs", [0, 1])
@pytest.mark.parametrize("N,KB", [(32, 1), (32, 2), (16, 3), (16, 1)])
def test_umma_known_answer(N, KB, a_in_regs):
    import torch
    from sparrowrecsys_b200 import _lib
    rng = np.random.default_rng(N * 10 + KB)
    K = 64 * KB
    A = rng.standard_normal((128, K)).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    dA, dB = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    dD = torch.zeros(128, N, dtype=torch.float32, device="cuda:0")
    _lib.check(_lib.load().srs_selftest_wgmma(dA.data_ptr(), dB.data_ptr(), dD.data_ptr(), N, KB,
                                              a_in_regs, 0))
    ref = _bf16_trunc(A).astype(np.float64) @ _bf16_trunc(B).astype(np.float64).T
    got = dD.cpu().numpy()
    err = np.abs(got - ref).max()
    assert err < 1e-4 * max(1.0, np.abs(ref).max()), "max err %g (N=%d KB=%d regsA=%d)" % (err, N, KB, a_in_regs)
