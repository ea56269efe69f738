"""din_wg_kernel at E <= 32 walks its rows in items of R = 2 rows at one chunk (csrc/din_wg.cu, DinWgLayout::R).  The GPU tests cover the edges where a
warpgroup's last item has fewer live rows than R: short last tiles, rows spanning several chunks, all-padding rows
beside full ones, and an out-of-range id in one row.  Checked against the float64 oracle with the tolerances of
tests/test_gpu_din_wg_groups.py, scores bit-identical under grid caps 1, 7 and 0 (GPU tests: pytest -m gpu).  The
CPU test compiles the default layout, held to zero spill bytes, and the one-row, five-warpgroup layout kept for
measurements (which spills a few bytes); neither may serialise its wgmma."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import ctr_oracle as O
from sparrowrecsys_b200 import build
from sparrowrecsys_b200.features import synthetic_features
from sparrowrecsys_b200.spec import baseline_spec, default_spec
from sparrowrecsys_b200.weights import init_weights

PROB_ATOL = 2e-5
LOGIT_ATOL = 2e-4


def _model(spec, W):
    from sparrowrecsys_b200.model import CTRModel
    return CTRModel(spec, W, device=0, options={"din_impl": "tc"})


def _check(spec, W, feats):
    with _model(spec, W) as m:
        assert m.kernel_name == "din_wg_kernel"
        p, z = m.predict_with_logits(feats)
        for n in (1, 7, 0):
            m.set_sm_limit(n)
            assert np.array_equal(m.predict(feats), p), n
    po, zo = O.forward(spec, W, feats)
    assert np.abs(z - zo).max() <= LOGIT_ATOL, "logit err %g" % np.abs(z - zo).max()
    assert np.abs(p - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p - po).max()
    return p


# B = 32 + r: the last tile has r rows, so with row pairs some warpgroup ends on a pair with one live row
@pytest.mark.gpu
@pytest.mark.parametrize("B", [32 + r for r in range(1, 9)] + [4095])
def test_last_pair_with_one_row_t50(B):
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 700 + B % 97)
    _check(spec, W, synthetic_features(spec, B, seed=700 + B))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [33, 35, 37, 39, 63, 70])
def test_last_pair_with_one_row_multi_chunk(B):
    """T = 129: a pair spans three items (the last of one position) while its second row is missing."""
    spec = default_spec("din", emb_dim=32, hist_len=129, n_movies=27279, n_users=5000)
    W = init_weights(spec, 800 + B)
    _check(spec, W, synthetic_features(spec, B, seed=800 + B))


@pytest.mark.gpu
@pytest.mark.parametrize("hist_len", [50, 129])
def test_all_padding_rows_paired_with_full_rows(hist_len):
    """Every other row's history is all padding (id 0 everywhere), the rows between them full."""
    spec = default_spec("din", emb_dim=32, hist_len=hist_len, n_movies=27279, n_users=5000)
    W = init_weights(spec, 900 + hist_len)
    B = 75
    feats = synthetic_features(spec, B, seed=900 + hist_len, pad_history=False)
    for k in range(1, hist_len + 1):
        col = np.asarray(feats["userRatedMovie%d" % k]).copy()
        col[0::2] = 0
        feats["userRatedMovie%d" % k] = col
    _check(spec, W, feats)


@pytest.mark.gpu
def test_out_of_range_id_in_one_row_of_a_pair():
    """An out-of-range history id in one row latches the error word; the other rows' scores do not change."""
    import torch
    from sparrowrecsys_b200.features import encode_batch
    spec = baseline_spec("cfg3_din")
    W = init_weights(spec, 41)
    B = 64
    feats = synthetic_features(spec, B, seed=41)
    bad_row = 4                       # at G = 4, R = 2 the second row of warpgroup 0's first pair
    with _model(spec, W) as m:
        ref = m.predict(feats)[:, 0]
        enc = encode_batch(spec, feats)
        enc.hist = np.array(enc.hist, copy=True)
        enc.hist[bad_row, 3] = spec.n_movies + 7
        out = torch.empty(B, dtype=torch.float32, device="cuda:0")
        m.predict_device(m.to_device(enc), out)
        with pytest.raises(ValueError):
            m.status()
        m.status()                    # cleared by the report
        got = out.cpu().numpy()
    keep = np.arange(B) != bad_row
    assert np.array_equal(got[keep], ref[keep])


@pytest.mark.parametrize("defines", [[], ["-DSRS_DIN_WG_ROWS32=1", "-DSRS_DIN_WG_GROUPS32=5"]],
                         ids=["default", "rows1_groups5"])
def test_layouts_compile_without_serialised_wgmma(defines):
    src = os.path.join(build.CSRC, "din_wg.cu")
    with tempfile.TemporaryDirectory(prefix="srs_din_wg_rows_") as tmp:
        cmd = [build.nvcc_path(), *build.ARCH, "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
               "--extended-lambda", *defines, "-Xptxas", "-v",
               "-c", src, "-o", os.path.join(tmp, "din_wg.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out
    assert "C7520" not in out, out    # no serialised wgmma
    found = {}
    for blk in re.split(r"Compiling entry function '", out)[1:]:
        m = re.search(r"din_wg_kernelILi(\d+)E", blk.split("'", 1)[0])
        if not m:
            continue
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", blk)
        assert spill, blk
        found[int(m.group(1))] = (int(spill.group(1)), int(spill.group(2)))
    assert sorted(found) == [32, 64], out
    for ep, (st, ld) in found.items():
        if defines and ep == 32:
            continue                  # the one-row layout at G = 5 (cap 102 registers) spills a few bytes
        assert st == 0 and ld == 0, "din_wg_kernel<%d> spills: %d bytes stored, %d loaded" % (ep, st, ld)
