"""BinaryClassificationMetrics on the device (csrc/binary_metrics.cu, sparrowrecsys_b200/evaluation.py) against the
float64 oracle in oracle/binary_metrics.py.

Counts, thresholds and every curve point are bit-equal to the oracle's (at beta 0, F-measure's 0 / 0 points are
NaN on both sides); each area lies within 1e-13 of the exactly
rounded sum (math.fsum) of the oracle's trapezoids.  Sizes run from 1 pair through the area kernel's 2048-point
chunk and the grid's edges to 10^6, and to 10^8 quantised scores on the device path.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import binary_metrics as BM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CHUNK = 2048                    # kChunk: points per block of bm_area_chunk_kernel
GRID = 256 * 132 * 64           # one full grid-stride pass of the 256-thread kernels (kMaxGridBlocks)
AREA_TOL = 1e-13


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def assert_set_matches(dev, k, want, beta=0.5):
    """Set k of the device metrics against the oracle's BinaryMetrics `want`."""
    sm = dev.summary(k)
    assert (sm.n, sm.positives, sm.negatives, sm.thresholds) == \
        (want.n, want.positives, want.negatives, want.thresholds().shape[0])
    tp, fp = dev.confusions(k)
    assert np.array_equal(tp, want.tp) and np.array_equal(fp, want.fp)
    for got, ref in ((dev.thresholds(k), want.thresholds()), (dev.roc(k), want.roc()), (dev.pr(k), want.pr()),
                     (dev.precision_by_threshold(k), want.precision_by_threshold()),
                     (dev.recall_by_threshold(k), want.recall_by_threshold()),
                     (dev.f_measure_by_threshold(1.0, k), want.f_measure_by_threshold(1.0)),
                     (dev.f_measure_by_threshold(beta, k), want.f_measure_by_threshold(beta))):
        assert got.shape == ref.shape and np.array_equal(_bits(got), _bits(ref))
    # at beta 0 a point with recall 0 < precision is 0 / 0: NaN on both sides, whose bit patterns differ
    got, ref = dev.f_measure_by_threshold(0.0, k), want.f_measure_by_threshold(0.0)
    nan = np.isnan(ref[:, 1])
    assert np.array_equal(np.isnan(got[:, 1]), nan) and np.array_equal(_bits(got[~nan]), _bits(ref[~nan]))
    assert abs(sm.area_under_roc - math.fsum(BM.trapezoid_terms(want.roc()))) <= AREA_TOL
    assert abs(sm.area_under_pr - math.fsum(BM.trapezoid_terms(want.pr()))) <= AREA_TOL


def check(scores, labels, num_bins=0, offsets=None):
    from sparrowrecsys_b200.evaluation import BinaryClassificationMetrics
    s, y = np.asarray(scores, np.float64), np.asarray(labels, np.float64)
    off = [0, s.shape[0]] if offsets is None else list(offsets)
    with BinaryClassificationMetrics(s, y, num_bins, offsets) as m:
        assert m.n_sets == len(off) - 1
        for k in range(len(off) - 1):
            assert_set_matches(m, k, BM.BinaryMetrics(s[off[k]:off[k + 1]], y[off[k]:off[k + 1]], num_bins))
        return [(m.area_under_roc(k), m.area_under_pr(k)) for k in range(len(off) - 1)]


def tied(n, seed, levels=None):
    """n scores with ties (float32-rounded, or drawn from `levels` distinct values) and 0/1 labels."""
    rng = np.random.default_rng(seed)
    if levels:
        s = (rng.integers(0, levels, n) / levels).astype(np.float64)
    else:
        s = rng.random(n).astype(np.float32).astype(np.float64)
    y = (rng.random(n) < 0.3 + 0.4 * s).astype(np.float64)
    return s, y


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 1, GRID - 1, GRID + 1,
                               10 ** 6])
def test_sizes_match_the_oracle(n):
    s, y = tied(n, n)
    check(s, y)
    if n >= CHUNK:
        check(*tied(n, n + 1, levels=CHUNK + 1))                 # thresholds around the chunk edge


@pytest.mark.gpu
@pytest.mark.parametrize("num_bins", [0, 1, 2, 3, 1000, 10 ** 6])
def test_num_bins(num_bins):
    s, y = tied(200_000, 3)
    check(s, y, num_bins)
    s, y = tied(20_000, 4, levels=4099)                            # grouping 1, 2, 3 and non-dividing counts
    check(s, y, num_bins)


@pytest.mark.gpu
def test_edge_inputs():
    nan2 = np.array([0xFFF8000000000001, 0x7FF0000000000001], np.uint64).view(np.float64)
    special = np.array([math.nan, nan2[0], nan2[1], 0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 1.0, -1.0])
    rng = np.random.default_rng(7)
    n = 50_000
    s = special[rng.integers(0, special.size, n)]
    y = rng.choice(np.array([0.0, 1.0, 0.3, 0.7, 0.5, math.nan, -2.0, 2.0]), n)
    for nb in (0, 1, 2, 3, 11, 12):
        check(s, y, nb)
    for case in [([0.4], [1]), ([0.4], [0]), ([-0.0, 0.0], [1, 0]), ([math.nan] * 3, [1, 0, 1]),
                 ([0.3, 0.7, 0.7], [0, 0, 0]), ([0.3, 0.7, 0.7], [1, 1, 1])]:
        for nb in (0, 1, 2):
            check(*case, num_bins=nb)


@pytest.mark.gpu
def test_batched_sets_equal_one_call_per_set():
    """Every set's counts and areas against the oracle; the curves of 1 and 2 sets, and of 40 sampled sets of 10^4,
    bit-equal to the oracle's and to a call of their own."""
    from sparrowrecsys_b200.evaluation import BinaryClassificationMetrics
    rng = np.random.default_rng(11)
    for n_sets in (1, 2, 10_000):
        sizes = rng.integers(1, 300, n_sets)
        sizes[:: 7] = 1
        if n_sets > 2:
            sizes[3] = 3 * CHUNK + 5
        off = np.concatenate([[0], np.cumsum(sizes)])
        s, y = tied(int(off[-1]), n_sets, levels=97)
        y[rng.random(y.size) < 0.05] = 0.7
        for nb in (0, 3):
            with BinaryClassificationMetrics(s, y, nb, off) as m:
                sample = set(rng.choice(n_sets, min(n_sets, 40), replace=False).tolist()) | {0, n_sets - 1}
                for k in range(n_sets):
                    want = BM.BinaryMetrics(s[off[k]:off[k + 1]], y[off[k]:off[k + 1]], nb)
                    if k in sample:
                        assert_set_matches(m, k, want)
                        with BinaryClassificationMetrics(s[off[k]:off[k + 1]], y[off[k]:off[k + 1]], nb) as one:
                            a, b = m.summary(k), one.summary()
                            assert (a.thresholds, a.area_under_roc, a.area_under_pr) == \
                                (b.thresholds, b.area_under_roc, b.area_under_pr)
                            assert np.array_equal(_bits(m.roc(k)), _bits(one.roc()))
                            assert np.array_equal(_bits(m.pr(k)), _bits(one.pr()))
                    else:
                        sm = m.summary(k)
                        assert (sm.n, sm.positives, sm.thresholds) == \
                            (want.n, want.positives, want.thresholds().shape[0])
                        assert abs(sm.area_under_roc - math.fsum(BM.trapezoid_terms(want.roc()))) <= AREA_TOL
                        assert abs(sm.area_under_pr - math.fsum(BM.trapezoid_terms(want.pr()))) <= AREA_TOL


@pytest.mark.gpu
def test_device_path_equals_host_path():
    import torch
    from sparrowrecsys_b200.evaluation import BinaryClassificationMetrics
    rng = np.random.default_rng(12)
    n = 300_001
    s32 = np.float32(rng.random(n) * 2 - 0.5)
    s32[:: 101] = np.float32(0.25)
    s32[5], s32[6], s32[7] = np.float32(np.nan), np.float32(-0.0), np.float32(0.0)
    y = rng.integers(-1, 3, n).astype(np.int32)
    off = np.array([0, 1, 1000, 1001, 250_000, n], np.int64)
    ds, dy = torch.from_numpy(s32).cuda(), torch.from_numpy(y).cuda()
    for nb in (0, 5):
        with BinaryClassificationMetrics(ds, dy, nb, off) as d, \
                BinaryClassificationMetrics(s32.astype(np.float64), y.astype(np.float64), nb, off) as h:
            for k in range(off.size - 1):
                a, b = d.summary(k), h.summary(k)
                assert (a.n, a.positives, a.thresholds, a.area_under_roc, a.area_under_pr) == \
                    (b.n, b.positives, b.thresholds, b.area_under_roc, b.area_under_pr)
                for f in ("roc", "pr", "thresholds", "precision_by_threshold", "recall_by_threshold"):
                    assert np.array_equal(_bits(getattr(d, f)(k)), _bits(getattr(h, f)(k))), f
                assert np.array_equal(d.confusions(k)[0], h.confusions(k)[0])
    with BinaryClassificationMetrics(ds, dy.to(torch.int64)) as d:         # integer labels of any width
        assert d.summary().positives == int((y > 0).sum())
    with pytest.raises(TypeError):
        BinaryClassificationMetrics(ds.double(), dy)
    with pytest.raises(TypeError):
        BinaryClassificationMetrics(ds, dy.float())


@pytest.mark.gpu
def test_two_calls_give_the_same_bits():
    from sparrowrecsys_b200.evaluation import BinaryClassificationMetrics
    s, y = tied(3_000_000, 21)
    off = np.array([0, 1_000_000, 1_000_001, 3_000_000], np.int64)
    runs = []
    for _ in range(2):
        with BinaryClassificationMetrics(s, y, 0, off) as m:
            runs.append([(m.area_under_roc(k), m.area_under_pr(k), _bits(m.roc(k)).tobytes()) for k in range(3)])
    assert runs[0] == runs[1]


@pytest.mark.gpu
def test_rejections_leave_nothing_allocated():
    import ctypes as C
    import torch
    from sparrowrecsys_b200 import _lib
    from sparrowrecsys_b200.evaluation import BinaryClassificationMetrics
    lib = _lib.load()
    s, y = tied(5000, 31)
    with BinaryClassificationMetrics(s, y) as m:                            # warm: context and module loaded
        T = m.summary().thresholds
    torch.cuda.synchronize()
    free0, launches0 = torch.cuda.mem_get_info()[0], lib.srs_launch_count()
    for kw in (dict(num_bins=-1), dict(set_offsets=[0, 10, 10, 5000]), dict(set_offsets=[0, 4999]),
               dict(set_offsets=[1, 5000])):
        with pytest.raises(ValueError):
            BinaryClassificationMetrics(s, y, **kw)
    with pytest.raises(ValueError):
        BinaryClassificationMetrics(s[:0], y[:0])
    with BinaryClassificationMetrics(s, y) as m:
        dst = np.full(2 * (T + 2), 3.0)
        for k, which in ((1, _lib.SRS_BM_ROC), (-1, _lib.SRS_BM_ROC), (0, 6), (0, -1)):
            rc = lib.srs_binary_metrics_curve(m._h, k, which, 1.0, dst.ctypes.data)
            assert rc == _lib.SRS_ERR_INVALID and np.all(dst == 3.0)
        out = _lib.SrsBinarySummary()
        assert lib.srs_binary_metrics_summary(m._h, 1, C.byref(out)) == _lib.SRS_ERR_INVALID
        with pytest.raises(ValueError):
            m.roc(1)
        launches1 = lib.srs_launch_count()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0
    assert launches1 > launches0


@pytest.mark.gpu
def test_1e8_quantised_scores_on_the_device_path():
    """10^8 pairs over 1001 float32 score levels, labels drawn with the level's probability, on the device path.
    The call's device memory peaks near 33 bytes a pair (two key and two tag buffers for the radix sort, run flags,
    cumulative counts and run starts): about 3.3 GB beside the 0.8 GB of inputs."""
    import torch
    from sparrowrecsys_b200.evaluation import BinaryClassificationMetrics
    n, L = 10 ** 8, 1001
    g = torch.Generator(device="cuda").manual_seed(5)
    idx = torch.randint(0, L, (n,), device="cuda", generator=g)
    levels = (torch.arange(L, device="cuda", dtype=torch.float64) / (L - 1)).float()
    s = levels[idx]
    y = (torch.rand(n, device="cuda", generator=g) < s).to(torch.int32)
    pos = torch.bincount(idx, weights=y.double(), minlength=L).cpu().numpy().astype(np.int64)
    cnt = torch.bincount(idx, minlength=L).cpu().numpy().astype(np.int64)
    keep = cnt > 0
    lv = levels.double().cpu().numpy()[keep][::-1]                         # threshold order: descending
    pos, neg = pos[keep][::-1], (cnt - pos)[keep][::-1]
    for nb in (0, 7):
        want = BM.BinaryMetrics.from_counts(lv, pos, neg, nb)
        with BinaryClassificationMetrics(s, y, nb) as m:
            assert_set_matches(m, 0, want)
    del idx, s, y
    torch.cuda.empty_cache()


# ---- end to end: neuralcf/002 on the reference's test rows ---------------------------------------------------
def _neuralcf_002():
    z = np.load(os.path.join(GOLDEN, "neuralcf_002_testset.npz"))
    W = {k.replace("__", "/"): z[k] for k in z.files
         if k not in ("user_ids", "user_rows", "movieId", "userId", "label")}
    table = np.zeros((30001, z["user_rows"].shape[1]), np.float32)
    table[z["user_ids"]] = z["user_rows"]
    W["userId_embedding"] = table
    return W, {"movieId": z["movieId"], "userId": z["userId"]}, z["label"].astype(np.int32)


@pytest.mark.gpu
def test_end_to_end_neuralcf_002(tmp_path):
    import json
    import torch
    from sparrowrecsys_b200.evaluation import BinaryClassificationEvaluator, BinaryClassificationMetrics, \
        evaluate, java_double
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.spec import default_spec
    with open(os.path.join(GOLDEN, "binary_metrics.json")) as f:
        ref = json.load(f)
    W, feats, y = _neuralcf_002()
    with CTRModel(default_spec("neuralcf"), W) as model:
        p = model.predict(feats)[:, 0]
    s = p.astype(np.float64)
    want = BM.BinaryMetrics(s, y)
    with BinaryClassificationMetrics(s, y) as m:
        assert_set_matches(m, 0, want)
        roc, pr = m.area_under_roc(), m.area_under_pr()
        assert (m.summary().n, m.summary().positives) == (ref["rows"], ref["positives"])
    assert abs(roc - ref["area_under_roc"]) <= 1e-6 and abs(pr - ref["area_under_pr"]) <= 1e-6
    with BinaryClassificationMetrics(torch.from_numpy(p).cuda(), torch.from_numpy(y).cuda()) as d:
        assert (d.area_under_roc(), d.area_under_pr()) == (roc, pr)
    assert BinaryClassificationEvaluator().evaluate(s, y) == roc
    assert BinaryClassificationEvaluator("areaUnderPR").evaluate(s, y) == pr
    assert evaluate(s, y) == (pr, roc)
    # the command line on a predictions CSV written from these scores
    csv = tmp_path / "predictions.csv"
    with open(csv, "w") as f:
        f.write("label,probability\n")
        f.writelines("%d,%r\n" % (a, b) for a, b in zip(y.tolist(), s.tolist()))
    r = subprocess.run([sys.executable, "-m", "sparrowrecsys_b200.evaluation", str(csv)], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert r.stdout.splitlines() == ["AUC under PR = " + java_double(pr), "AUC under ROC = " + java_double(roc)]
