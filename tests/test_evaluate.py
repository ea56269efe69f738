"""`model.evaluate`: Keras's loss, accuracy and ROC / PR AUC over labelled batches (csrc/metrics.cu,
srs_metrics_* and srs_evaluate_host_batches in csrc/model.cu, `CTRModel.evaluate`, `Metrics`).

* CPU: the restatement in oracle/keras_eval.py - thresholds, the bin-histogram formulation the kernel uses
  against the literal [n, 200] comparison, the AUCs against sklearn and hand-worked cases, the logit-path
  loss - the known-answer fixture of the shipped neuralcf/002 weights, and the srs_eval_result layout.
* GPU (pytest -m gpu): exact counts on crafted device buffers, determinism, every model kind against the
  oracle on the GPU's own scores, the known answer, errors, mixed call sequences, CUDA graphs, threads.
"""
import ctypes as C
import json
import os
import re
import threading

import numpy as np
import pytest

from oracle import ctr_oracle as O
from oracle import keras_eval as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
P_TOL = 2e-5              # GPU vs float64 oracle on probabilities (test_gpu_kernel_matrix.py)
LOSS_RTOL = 1e-6
CSRC_TILE = 1024          # rows per CTA of metrics_update_kernel (kMetRowsPerCta)
CSRC_MAX_CTAS = 264       # kMetMaxCtas


def adversarial_probs():
    """Every threshold, its float32 neighbours on both sides, 0, 0.5 with its neighbours, and 1."""
    t = K.keras_thresholds()
    vals = [t, np.nextafter(t, np.float32(-np.inf)), np.nextafter(t, np.float32(np.inf)),
            np.array([0.0, 0.5, 1.0], np.float32),
            np.nextafter(np.float32([0.5, 0.5]), np.float32([-np.inf, np.inf]))]
    p = np.concatenate(vals).astype(np.float32)
    return p[(p >= 0) & (p <= 1)]


def bin_counts(p, labels):
    """The kernel's formulation: bin k = #{j : p > t_j}, a (label, bin) histogram, TP / FP by suffix sums."""
    t = K.keras_thresholds()
    k = np.searchsorted(t, np.asarray(p, np.float32), side="left")          # #{t_j < p}
    pos = np.asarray(labels) != 0
    h1 = np.bincount(k[pos], minlength=201)
    h0 = np.bincount(k[~pos], minlength=201)
    tp = np.array([h1[j + 1:].sum() for j in range(200)], np.int64)
    fp = np.array([h0[j + 1:].sum() for j in range(200)], np.int64)
    return tp, fp, int((~pos).sum()) - fp, int(pos.sum()) - tp


def load_testset():
    z = np.load(os.path.join(GOLDEN, "neuralcf_002_testset.npz"))
    W = {k.replace("__", "/"): z[k] for k in z.files
         if k not in ("user_ids", "user_rows", "movieId", "userId", "label")}
    table = np.zeros((30001, z["user_rows"].shape[1]), np.float32)
    table[z["user_ids"]] = z["user_rows"]
    W["userId_embedding"] = table
    feats = {"movieId": z["movieId"], "userId": z["userId"], "label": z["label"]}
    with open(os.path.join(GOLDEN, "neuralcf_002_eval.json")) as f:
        ref = json.load(f)
    return W, feats, ref


# ---- CPU ----------------------------------------------------------------------------------------------
def test_thresholds_are_the_float32_images_of_keras_list():
    t = K.keras_thresholds()
    assert t.dtype == np.float32 and t.shape == (200,)
    assert t[0] == np.float32(-1e-7) and t[-1] == np.float32(1 + 1e-7)
    assert np.array_equal(t[1:-1], np.array([(i + 1) * 1.0 / 199 for i in range(198)]).astype(np.float32))
    assert np.all(np.diff(t) > 0)


def test_bin_histogram_equals_broadcast_comparison_on_adversarial_probabilities():
    p = adversarial_probs()
    rng = np.random.default_rng(0)
    for labels in (rng.integers(0, 2, p.shape[0]), np.ones(p.shape[0], int), np.zeros(p.shape[0], int)):
        got, want = bin_counts(p, labels), K.confusion_counts(p, labels)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
    # the neighbours really do land on both sides of their threshold
    t = K.keras_thresholds()
    assert np.all(np.nextafter(t[1:-1], np.float32(2)) > t[1:-1])


def test_roc_auc_matches_sklearn_on_one_score_per_bin():
    from sklearn.metrics import roc_auc_score
    t = K.keras_thresholds().astype(np.float64)
    mids = ((t[:-1] + t[1:]) / 2).astype(np.float32)               # one distinct score per bin
    rng = np.random.default_rng(1)
    for n in (50, 1000, 20000):
        p = mids[rng.integers(0, mids.shape[0], n)]
        lab = (rng.random(n) < 0.2 + 0.6 * p).astype(np.int32)
        r = K.keras_evaluate(p, np.zeros(n, np.float32), lab)
        assert abs(r["roc_auc"] - roc_auc_score(lab, p)) <= 1e-12


def test_auc_hand_worked_cases():
    z = np.zeros(4, np.float32)
    perfect = K.keras_evaluate(np.float32([0.1, 0.9]), z[:2], [0, 1])
    assert perfect["roc_auc"] == 1.0 and perfect["pr_auc"] == 1.0
    # single class: ROC AUC 0.0 (recall or fpr is div_no_nan(0, 0) everywhere).  PR: no positives -> 0.0;
    # only positives -> precision 1 at every step, each of the 4 steps adds slope 1 * dtp 1 / 4 -> 1.0
    r = K.keras_evaluate(np.float32([0.2, 0.4, 0.6, 0.8]), z, [0, 0, 0, 0])
    assert r["roc_auc"] == 0.0 and r["pr_auc"] == 0.0
    r = K.keras_evaluate(np.float32([0.2, 0.4, 0.6, 0.8]), z, [1, 1, 1, 1])
    assert r["roc_auc"] == 0.0 and r["pr_auc"] == 1.0
    # p = 0.2 0.4 0.6 0.8, labels 0 1 0 1.  (fpr, recall) by threshold band: (1,1) (.5,1) (.5,.5) (0,.5) (0,0)
    # -> ROC = .5*1 + .5*.5 = 0.75.  PR: predicted positives p = 4 3 2 1 0, tp = 2 2 1 1 0; the steps with
    # dtp = 1 are 3->2 (slope 1, intercept -1, ratio 3/2: (1 - ln 1.5) / 2) and 1->0 (slope 1, intercept 0: 1/2)
    r = K.keras_evaluate(np.float32([0.2, 0.4, 0.6, 0.8]), z, [0, 1, 0, 1])
    assert abs(r["roc_auc"] - 0.75) < 1e-15
    assert abs(r["pr_auc"] - (1 - np.log(1.5) / 2)) < 1e-15
    assert r["correct"] == 2 and r["accuracy"] == 0.5


def test_accuracy_counts_one_half_as_negative():
    r = K.keras_evaluate(np.float32([0.5, 0.5, np.nextafter(np.float32(0.5), np.float32(1))]),
                         np.zeros(3, np.float32), [0, 1, 1])
    assert r["correct"] == 2


def test_loss_takes_the_logit_path():
    logits = np.float32([30.0, -30.0])
    probs = np.float32(1 / (1 + np.exp(-logits.astype(np.float64))))
    r = K.keras_evaluate(probs, logits, [0, 1])
    assert abs(r["loss"] - 30.0) < 1e-5
    assert abs(K.clipped_bce(probs, [0, 1]).mean() - 16.118) < 1e-3       # what clipping would have given


def test_oracle_rejects_bad_inputs():
    z = np.zeros(2, np.float32)
    for p in ([0.2, np.nan], [0.2, 1.5], [-0.1, 0.2]):
        with pytest.raises(ValueError):
            K.keras_evaluate(np.float32(p), z, [0, 1])
    for lab in ([0, 2], [-1, 0]):
        with pytest.raises(ValueError):
            K.keras_evaluate(np.float32([0.2, 0.3]), z, lab)


def test_fixture_reproduces_its_json_and_the_whole_file_accuracy():
    from sparrowrecsys_b200.spec import default_spec
    W, feats, ref = load_testset()
    assert feats["label"].shape == (22440,) and np.unique(feats["userId"]).shape == (12146,)
    p, z = O.forward(default_spec("neuralcf"), W, {"movieId": feats["movieId"], "userId": feats["userId"]})
    r = K.keras_evaluate(p[:, 0], z[:, 0], feats["label"])
    for k in ("rows", "positives", "correct"):
        assert r[k] == ref[k]
    for k in ("tp", "fp", "tn", "fn"):
        assert r[k].tolist() == ref[k]
    for k in ("loss", "accuracy", "roc_auc", "pr_auc"):
        assert abs(r[k] - ref[k]) <= 1e-12, k
    with open(os.path.join(GOLDEN, "full_file_stats.json")) as f:
        stats = json.load(f)
    assert r["accuracy"] == stats["accuracy"] and abs(stats["accuracy"] - 0.678788) < 1e-6
    assert abs(ref["exact_rank_roc_auc"] - stats["roc_auc"]) < 1e-12


def test_eval_result_struct_matches_the_header():
    from sparrowrecsys_b200 import _lib
    with open(os.path.join(ROOT, "include", "srs_ctr.h")) as f:
        text = f.read()
    body = re.search(r"typedef struct srs_eval_result \{(.*?)\} srs_eval_result;", text, re.S).group(1)
    fields = []
    for ctype, names in re.findall(r"(int64_t|double)\s+([^;]+);", body):
        fields += [(n.strip(), ctype) for n in names.split(",")]
    want = {"int64_t": C.c_int64, "double": C.c_double}
    assert [(n, want[t]) for n, t in fields] == list(_lib.SrsEvalResult._fields_)
    assert C.sizeof(_lib.SrsEvalResult) == 56


# ---- GPU ----------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def device_metrics(probs, logits, labels, chunks=None):
    """Fold the rows through srs_metrics_update_device (in `chunks` updates) and return the result dict."""
    from sparrowrecsys_b200.model import Metrics
    n = probs.shape[0]
    bounds = chunks or [(0, n)]
    P, L, Y = _dev(np.float32(probs)), _dev(np.float32(logits)), _dev(np.int32(labels))
    with Metrics(0) as mt:
        for lo, hi in bounds:
            mt.update_device(P[lo:hi], L[lo:hi], Y[lo:hi])
        return mt.result()


def assert_matches_oracle(got, want, loss_rtol=LOSS_RTOL):
    for k in ("rows", "positives", "correct"):
        assert got[k] == want[k], k
    for k in ("tp", "fp", "tn", "fn"):
        assert np.array_equal(np.asarray(got[k]), want[k]), k
    assert abs(got["loss"] - want["loss"]) <= loss_rtol * abs(want["loss"])
    assert got["accuracy"] == want["accuracy"]
    assert abs(got["roc_auc"] - want["roc_auc"]) <= 1e-12
    assert abs(got["pr_auc"] - want["pr_auc"]) <= 1e-12


def crafted(n, seed):
    """n rows cycling through the adversarial probabilities, logits up to +-30, labels 0/1."""
    rng = np.random.default_rng(seed)
    adv = adversarial_probs()
    p = np.concatenate([adv, rng.random(max(n - adv.shape[0], 0)).astype(np.float32)])[:n]
    p = p[rng.permutation(n)] if n > 1 else p
    x = rng.uniform(-30, 30, n).astype(np.float32)
    y = rng.integers(0, 2, n).astype(np.int32)
    return p, x, y


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 31, 33, CSRC_TILE - 1, CSRC_TILE, CSRC_TILE + 1,
                               CSRC_TILE * CSRC_MAX_CTAS - 1, CSRC_TILE * CSRC_MAX_CTAS + 1, 10 ** 6 + 1])
def test_device_update_exact_counts(n):
    p, x, y = crafted(n, n)
    assert_matches_oracle(device_metrics(p, x, y), K.keras_evaluate(p, x, y))


@pytest.mark.gpu
def test_device_update_adversarial_values_all_labels():
    p = adversarial_probs()
    x = np.linspace(-30, 30, p.shape[0]).astype(np.float32)
    for y in (np.zeros(p.shape[0], np.int32), np.ones(p.shape[0], np.int32),
              (np.arange(p.shape[0]) % 2).astype(np.int32)):
        assert_matches_oracle(device_metrics(p, x, y), K.keras_evaluate(p, x, y))


@pytest.mark.gpu
def test_device_update_clustered_scores():
    """Many rows of one warp in one bin: the warp-aggregated shared atomics."""
    n = 100_000
    rng = np.random.default_rng(5)
    p = np.float32(rng.choice(np.float32([0.3, 0.3000001, 0.7]), n))
    x, y = rng.normal(size=n).astype(np.float32), rng.integers(0, 2, n).astype(np.int32)
    assert_matches_oracle(device_metrics(p, x, y), K.keras_evaluate(p, x, y))


@pytest.mark.gpu
def test_device_update_deterministic_and_split_invariant():
    n = 300_001
    p, x, y = crafted(n, 7)
    a = device_metrics(p, x, y)
    b = device_metrics(p, x, y)
    assert a["loss"] == b["loss"] and a["pr_auc"] == b["pr_auc"] and a["roc_auc"] == b["roc_auc"]
    cuts = [0, 1, 4096, 77777, 270336, n]
    c = device_metrics(p, x, y, chunks=list(zip(cuts[:-1], cuts[1:])))
    for k in ("rows", "positives", "correct", "accuracy", "roc_auc", "pr_auc"):
        assert c[k] == a[k]
    for k in ("tp", "fp", "tn", "fn"):
        assert np.array_equal(c[k], a[k])
    assert abs(c["loss"] - a["loss"]) <= 1e-12 * abs(a["loss"])


@pytest.mark.gpu
def test_device_update_errors_latch_until_reset():
    import torch
    from sparrowrecsys_b200.model import Metrics
    with Metrics(0) as mt:
        for p, y in (([0.2, np.nan], [0, 1]), ([0.2, 1.5], [0, 1]), ([0.2, 0.3], [0, 2]), ([0.2, 0.3], [-1, 0])):
            mt.reset()
            mt.update_device(_dev(np.float32(p)), _dev(np.float32([0, 0])), _dev(np.int32(y)))
            with pytest.raises(ValueError):
                mt.result()
        mt.reset()
        with pytest.raises(ValueError):                 # no rows
            mt.result()
        mt.update_device(_dev(np.float32([0.2, 0.7])), _dev(np.float32([0, 0])), _dev(np.int32([0, 1])))
        assert mt.result()["correct"] == 2
        with pytest.raises(ValueError):
            mt.update_device(_dev(np.float32([0.2])), _dev(np.float32([0, 0])), _dev(np.int32([0])))
        torch.cuda.synchronize()


# ---- every model kind ----------------------------------------------------------------------------------
def _cases():
    from sparrowrecsys_b200.spec import default_spec
    small = dict(n_movies=3000, n_users=4000)
    return [
        ("embeddingmlp_tc", default_spec("embeddingmlp", **small), {}, "embmlp_tc_kernel"),
        ("embeddingmlp_cc", default_spec("embeddingmlp", **small), {"embmlp_impl": "cudacore"}, "embmlp_kernel"),
        ("widendeep", default_spec("widendeep", **small), {}, "embmlp_tc_kernel<wide&deep>"),
        ("neuralcf", default_spec("neuralcf", **small), {}, None),
        ("twotowers_dense", default_spec("twotowers", final_dense=True, **small), {}, None),
        ("deepfm_tc", default_spec("deepfm", emb_dim=16, **small), {}, "deepfm_tc_kernel"),
        ("deepfm_cc", default_spec("deepfm", **small), {"deepfm_impl": "cudacore"}, None),
        ("deepfm_v2", default_spec("deepfm_v2", **small), {}, None),
        ("din_wg", default_spec("din", emb_dim=32, hist_len=50, **small), {}, "din_wg_kernel"),
        ("din_cc", default_spec("din", emb_dim=32, hist_len=50, **small), {"din_impl": "cudacore"}, "din_kernel"),
        ("din_narrow", default_spec("din", emb_dim=32, hist_len=50, **small), {"narrow": True}, "din_wg_kernel"),
    ]


CASE_IDS = [c[0] for c in _cases()]


def _labelled(spec, n, seed, p=None):
    from sparrowrecsys_b200.features import synthetic_features
    feats = synthetic_features(spec, n, seed=seed)
    rng = np.random.default_rng(seed + 1)
    feats["label"] = (rng.random(n) < (0.5 if p is None else p)).astype(np.int32)
    return feats


def _near(p64, tol=P_TOL):
    marks = np.concatenate([K.keras_thresholds().astype(np.float64), [0.5]])
    idx = np.searchsorted(marks, p64)
    d = np.minimum(np.abs(p64 - marks[np.clip(idx, 0, marks.shape[0] - 1)]),
                   np.abs(p64 - marks[np.clip(idx - 1, 0, marks.shape[0] - 1)]))
    return int((d <= tol).sum())


def _model(spec, opts, seed=0):
    from sparrowrecsys_b200.model import CTRModel
    from sparrowrecsys_b200.weights import init_weights
    opts = dict(opts)
    narrow = opts.pop("narrow", False)
    W = init_weights(spec, seed)
    return CTRModel(spec, W, narrow_ids=narrow, options=opts), W


def _result_dict(r):
    return {k: getattr(r, k) for k in ("rows", "positives", "correct", "loss", "accuracy", "roc_auc", "pr_auc")}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASE_IDS)
def test_evaluate_every_model_kind(case):
    name, spec, opts, kernel = [c for c in _cases() if c[0] == case][0]
    m, W = _model(spec, opts, seed=3)
    with m:
        if kernel:
            assert m.kernel_name == kernel
        n = 5000
        feats = _labelled(spec, n, seed=11)
        p, z = m.predict_with_logits(feats)
        want = K.keras_evaluate(p[:, 0], z[:, 0], feats["label"])
        for bs in (None, 777):
            got = _result_dict(m.evaluate_result(feats, batch_size=bs))
            for k in ("rows", "positives", "correct", "accuracy", "roc_auc", "pr_auc"):
                assert got[k] == pytest.approx(want[k], abs=1e-12, rel=0), k
            assert abs(got["loss"] - want["loss"]) <= LOSS_RTOL * want["loss"]
        loss, acc, roc, pr = m.evaluate(feats)
        assert (acc, roc, pr) == (got["accuracy"], got["roc_auc"], got["pr_auc"])
        # against the float64 oracle forward: counts move by at most the rows near a threshold or 0.5
        p64, z64 = O.forward(spec, W, feats, dtype=np.float64)
        ref = K.keras_evaluate(np.clip(p64[:, 0], 0, 1), z64[:, 0], feats["label"])
        near = _near(p64[:, 0])
        for k in ("tp", "fp", "tn", "fn"):
            assert np.abs(want[k] - ref[k]).max() <= near, (k, near)
        assert abs(want["correct"] - ref["correct"]) <= near


# ---- known answer ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_neuralcf_002_known_answer():
    import tfrecmodel.neuralcf as ncf
    W, feats, ref = load_testset()
    ncf.load(W)
    try:
        r12 = ncf.model.evaluate_result(feats, batch_size=12)          # Keras's batch, 1870 batches
        r1 = ncf.model.evaluate_result(feats)                          # one batch
        assert ncf.evaluate(feats, batch_size=12) == (r12.loss, r12.accuracy, r12.roc_auc, r12.pr_auc)
    finally:
        ncf.model.close()
        ncf.model = None
    n, r = ref["rows"], ref["near"]
    P, N = ref["positives"], n - ref["positives"]
    for res in (r12, r1):
        assert res.rows == n and res.positives == P
        assert abs(res.accuracy - 0.678788) <= r / n + 1e-6
        assert abs(res.accuracy - ref["accuracy"]) <= r / n
        # moving one row to a neighbouring bin changes one point of the curves by 1/P or 1/N
        assert abs(res.roc_auc - ref["roc_auc"]) <= r * (1 / P + 1 / N)
        assert abs(res.pr_auc - ref["pr_auc"]) <= r * 2 / P
        assert abs(res.loss - ref["loss"]) <= 1e-5 * ref["loss"]
    for k in ("rows", "positives", "correct", "accuracy", "roc_auc", "pr_auc"):
        assert getattr(r12, k) == getattr(r1, k), k
    assert abs(r12.loss - r1.loss) <= 1e-12 * r1.loss


# ---- errors ----------------------------------------------------------------------------------------------
def _clean_after(m, feats, want_p):
    assert np.array_equal(m.predict(feats), want_p)
    m.status()


@pytest.mark.gpu
def test_evaluate_errors_leave_the_model_clean():
    from sparrowrecsys_b200.spec import default_spec
    spec = default_spec("widendeep", n_movies=3000, n_users=4000)
    m, _ = _model(spec, {})
    with m:
        feats = _labelled(spec, 3000, seed=2)
        want_p = m.predict(feats)
        good = m.evaluate(feats, batch_size=1000)
        bad_id = dict(feats, movieId=feats["movieId"].copy())
        bad_id["movieId"][1234] = spec.n_movies
        with pytest.raises(ValueError):
            m.evaluate(bad_id, batch_size=1000)
        _clean_after(m, feats, want_p)
        for v in (2, -1):
            lab = feats["label"].copy()
            lab[2999] = v
            with pytest.raises(ValueError, match="label"):
                m.evaluate(feats, labels=lab, batch_size=1000)
            _clean_after(m, feats, want_p)
        with pytest.raises(ValueError):
            m.evaluate({k: v[:0] for k, v in feats.items()})
        with pytest.raises(KeyError):
            m.evaluate({k: v for k, v in feats.items() if k != "label"})
        _clean_after(m, feats, want_p)
        assert m.evaluate(feats, batch_size=1000) == good
    # a NaN numeric: DeepFM_v2 adds the numerics' first-order term straight to the logit (a ReLU layer, as in
    # Wide&Deep, would turn the NaN into 0)
    v2 = default_spec("deepfm_v2", n_movies=3000, n_users=4000)
    m, _ = _model(v2, {})
    with m:
        feats = _labelled(v2, 3000, seed=5)
        want_p = m.predict(feats)
        nan = dict(feats, movieAvgRating=np.asarray(feats["movieAvgRating"], np.float32).copy())
        nan["movieAvgRating"][17] = np.nan
        assert np.isnan(m.predict(nan)[17, 0])
        with pytest.raises(ValueError, match="probability"):
            m.evaluate(nan, batch_size=1000)
        _clean_after(m, feats, want_p)
    tt = default_spec("twotowers", hidden=(10,), final_dense=False, n_movies=3000, n_users=4000)
    m, _ = _model(tt, {})
    with m:
        feats = _labelled(tt, 100, seed=3)
        want_p = m.predict(feats)
        with pytest.raises(ValueError, match="raw dot"):
            m.evaluate(feats)
        _clean_after(m, feats, want_p)
    dn = default_spec("dien", n_movies=3000, n_users=4000)
    m, _ = _model(dn, {})
    with m:
        feats = _labelled(dn, 100, seed=4)
        want_p = m.predict(feats)
        with pytest.raises(ValueError, match="DIEN"):
            m.evaluate(feats)
        _clean_after(m, feats, want_p)
    import tfrecmodel.dien as D
    with pytest.raises(NotImplementedError, match="auxiliary"):
        D.evaluate(feats)


# ---- mixed sequences, graphs, threads ---------------------------------------------------------------------
@pytest.mark.gpu
def test_evaluate_interleaved_with_every_host_entry_point():
    from sparrowrecsys_b200.features import encode_batch
    from sparrowrecsys_b200.spec import default_spec
    spec = default_spec("neuralcf", n_movies=3000, n_users=4000)
    m, W = _model(spec, {}, seed=9)
    fresh, _ = _model(spec, {}, seed=9)
    with m, fresh:
        for step, n in enumerate((10, 700, 1025, 5000, 20000)):
            feats = _labelled(spec, n, seed=100 + step)
            bs = max(n // 3, 1)
            want_eval = fresh.evaluate(feats, batch_size=bs)
            want_p = fresh.predict(feats)
            assert m.evaluate(feats, batch_size=bs) == want_eval
            assert np.array_equal(m.predict(feats), want_p)
            assert m.evaluate(feats) == fresh.evaluate(feats)
            enc = encode_batch(spec, feats)
            keep, outs = [], []
            from sparrowrecsys_b200.model import _host_struct
            for slot in range(m.num_slots()):
                lo, hi = slot * n // 4, (slot + 1) * n // 4
                if hi == lo:
                    continue
                out = np.empty(hi - lo, np.float32)
                outs.append((lo, hi, out))
                m.submit_host(slot, _host_struct(enc.slice(lo, hi), keep), out.ctypes.data)
            assert m.evaluate(feats, batch_size=bs) == want_eval
            for slot in range(m.num_slots()):
                m.wait(slot)
            for lo, hi, out in outs:
                assert np.array_equal(out, want_p[lo:hi, 0])
            assert np.array_equal(m.predict(feats, batch_size=bs), want_p)
            idx, top, sc = m.rank_user(int(feats["userId"][0]), {}, feats["movieId"], 10, return_scores=True)
            assert m.evaluate(feats, batch_size=bs) == want_eval
            m.status()


@pytest.mark.gpu
def test_evaluate_under_sm_limits_and_after_slot_growth():
    from sparrowrecsys_b200.spec import baseline_spec
    spec = baseline_spec("cfg3_din")
    m, _ = _model(spec, {}, seed=4)
    with m:
        feats = _labelled(spec, 9000, seed=21)
        base = m.evaluate(feats, batch_size=1000)
        for lim in (8, 33, 0):
            m.set_sm_limit(lim)
            assert m.evaluate(feats, batch_size=1000) == base
        m.predict(feats, batch_size=4500)                 # other slot sizes and interleavings
        assert m.evaluate(feats, batch_size=1000) == base
        r7 = m.evaluate_result(feats, batch_size=700)
        r1 = m.evaluate_result(feats)
        assert (r7.correct, r7.roc_auc, r7.pr_auc) == (r1.correct, r1.roc_auc, r1.pr_auc)
        assert abs(r7.loss - r1.loss) <= 1e-12 * r1.loss
        assert (r1.accuracy, r1.roc_auc, r1.pr_auc) == base[1:]


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["din", "neuralcf"])
def test_cuda_graph_of_predict_and_metrics_update(model):
    import torch
    from sparrowrecsys_b200.model import Metrics
    from sparrowrecsys_b200.spec import baseline_spec, default_spec
    spec = baseline_spec("cfg3_din") if model == "din" else default_spec("neuralcf", n_movies=3000, n_users=4000)
    m, _ = _model(spec, {}, seed=6)
    B, reps = 4096, 5
    with m, Metrics(0) as mt:
        feats = _labelled(spec, B, seed=31)
        db = m.to_device(feats)
        probs = torch.empty(B, device="cuda", dtype=torch.float32)
        logits = torch.empty_like(probs)
        lab = _dev(feats["label"].astype(np.int32))
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            m.predict_device(db, probs, logits, stream=s)
            mt.update_device(probs, logits, lab, stream=s)
        s.synchronize()
        once = mt.result()
        mt.reset(stream=s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            m.predict_device(db, probs, logits, stream=s)
            mt.update_device(probs, logits, lab, stream=s)
        torch.cuda.synchronize()
        mt.reset()
        torch.cuda.synchronize()
        for _ in range(reps):
            g.replay()
        rep = mt.result()
        for k in ("tp", "fp", "tn", "fn"):
            assert np.array_equal(rep[k], reps * once[k])
        assert rep["correct"] == reps * once["correct"] and rep["rows"] == reps * B
        assert abs(rep["loss"] - once["loss"]) <= 1e-12 * once["loss"]
        assert (rep["accuracy"], rep["roc_auc"], rep["pr_auc"]) == (once["accuracy"], once["roc_auc"], once["pr_auc"])
        want = K.keras_evaluate(probs.cpu().numpy(), logits.cpu().numpy(), feats["label"])
        assert once["correct"] == want["correct"] and np.array_equal(once["tp"], want["tp"])
        m.status()


@pytest.mark.gpu
def test_two_threads_evaluate_one_model():
    from sparrowrecsys_b200.spec import default_spec
    spec = default_spec("deepfm", emb_dim=16, n_movies=3000, n_users=4000)
    m, _ = _model(spec, {}, seed=8)
    with m:
        data = [_labelled(spec, 3000 + 1000 * i, seed=40 + i) for i in range(2)]
        serial = [m.evaluate(f, batch_size=500) for f in data]
        got = [[], []]

        def run(i):
            for _ in range(5):
                got[i].append(m.evaluate(data[i], batch_size=500))
        th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for i in range(2):
            assert got[i] == [serial[i]] * 5
        m.status()
