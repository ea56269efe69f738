"""mllib's BinaryClassificationMetrics restated in oracle/binary_metrics.py, checked without a device.

* Hand-worked known answers (one to six pairs: ties, one class, NaN, +-0, labels 0.3 / 0.7, binning), and the
  deliberate mistakes they must catch.
* An independent identity: the ROC area is the Mann-Whitney statistic under Spark's key order.
* Binning against a literal restatement of Spark's grouped(grouping) loop.
* The known answer of neuralcf/002 on the reference's test rows (binary_metrics.json).
* The C ABI's rejections, which come before any device call, and the Python front end's pure helpers.
"""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

from oracle import binary_metrics as BM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NAN2 = np.array([0xFFF8000000000001], np.uint64).view(np.float64)[0]     # a NaN with the sign bit and a payload

# (scores, labels, numBins, thresholds, TP, FP, area under ROC, area under PR)
KNOWN = [
    ([0.4], [1], 0, [0.4], [1], [0], 1.0, 1.0),
    ([0.4], [0], 0, [0.4], [0], [1], 0.0, 0.0),
    # ROC (0,0) (0,.5) (.5,.5) (.5,1) (1,1) (1,1); PR (0,1) (.5,1) (.5,.5) (1,2/3) (1,.5)
    ([0.2, 0.4, 0.6, 0.8], [0, 1, 0, 1], 0, [0.8, 0.6, 0.4, 0.2], [1, 1, 2, 2], [0, 1, 1, 2], 0.75, 0.5 + 7 / 24),
    # ties: 0.5 holds two positives and a negative; PR starts at (0, 2/3)
    ([0.5, 0.5, 0.1, 0.5], [1, 0, 0, 1], 0, [0.5, 0.1], [2, 2], [1, 2], 0.75, 2 / 3),
    # one class: no positive -> recall 0 everywhere, precision 0; no negative -> FPR 0, the (1,1) segment is all
    ([0.3, 0.7], [0, 0], 0, [0.7, 0.3], [0, 0], [1, 2], 0.0, 0.0),
    ([0.3, 0.7], [1, 1], 0, [0.7, 0.3], [1, 2], [0, 0], 1.0, 1.0),
    # every NaN is one threshold and it comes first
    ([0.1, math.nan, 0.9, NAN2], [0, 0, 1, 1], 0, [math.nan, 0.9, 0.1], [1, 2, 2], [1, 1, 2], 0.625, 0.25 + 7 / 24),
    # 0.0 and -0.0 are two thresholds, 0.0 above
    ([-0.0, 0.0], [1, 0], 0, [0.0, -0.0], [0, 1], [1, 1], 0.0, 0.25),
    # label > 0.5 is a positive: 0.3 and 0.5 and NaN are negatives, 0.7 a positive
    ([0.9, 0.2, 0.6, 0.1, 0.3, 0.4], [0.3, 0.7, 0.5, math.nan, 0.7, 2.0], 0,
     [0.9, 0.6, 0.4, 0.3, 0.2, 0.1], [0, 0, 1, 2, 3, 3], [1, 2, 2, 2, 2, 3], 1 / 3, None),
    # numBins 2 over 5 thresholds: grouping 2, runs {.9 .8} {.7 .6} {.5}, each at its first score
    ([0.9, 0.8, 0.7, 0.6, 0.5], [1, 0, 1, 0, 1], 2, [0.9, 0.7, 0.5], [1, 2, 3], [1, 2, 2], None, None),
    # numBins 3 over 5: grouping 1 < 2, no binning
    ([0.9, 0.8, 0.7, 0.6, 0.5], [1, 0, 1, 0, 1], 3, [0.9, 0.8, 0.7, 0.6, 0.5], [1, 1, 2, 2, 3], [0, 1, 1, 2, 2],
     None, None),
]


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and \
        np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)]) and \
        np.array_equal(np.signbit(a[a == 0]), np.signbit(b[b == 0]))


def known_answer_failures():
    bad = []
    for i, (s, y, nb, thr, tp, fp, roc, pr) in enumerate(KNOWN):
        m = BM.BinaryMetrics(np.array(s, np.float64), np.array(y, np.float64), nb)
        if not (_same(m.thresholds(), thr) and np.array_equal(m.tp, tp) and np.array_equal(m.fp, fp)):
            bad.append((i, "counts"))
        elif roc is not None and abs(m.area_under_roc() - roc) > 1e-15:
            bad.append((i, "roc", m.area_under_roc()))
        elif pr is not None and abs(m.area_under_pr() - pr) > 1e-15:
            bad.append((i, "pr", m.area_under_pr()))
    return bad


def test_hand_worked_known_answers():
    assert known_answer_failures() == []


def test_hand_worked_curves():
    m = BM.BinaryMetrics([0.2, 0.4, 0.6, 0.8], [0, 1, 0, 1])
    assert m.roc().tolist() == [[0, 0], [0, .5], [.5, .5], [.5, 1], [1, 1], [1, 1]]
    assert m.pr().tolist() == [[0, 1], [.5, 1], [.5, .5], [1, 2 / 3], [1, .5]]
    assert m.precision_by_threshold().tolist() == [[.8, 1], [.6, .5], [.4, 2 / 3], [.2, .5]]
    assert m.recall_by_threshold()[:, 1].tolist() == [.5, .5, 1, 1]
    f1 = m.f_measure_by_threshold()[:, 1]
    assert f1.tolist() == [2 * (1 * .5 / 1.5), 2 * (.25 / 1), 2 * ((2 / 3) / (2 / 3 + 1)), 2 * (.5 / 1.5)]
    f2 = BM.BinaryMetrics([0.3, 0.7], [0, 0]).f_measure_by_threshold(2.0)
    assert f2[:, 1].tolist() == [0.0, 0.0]                                   # p + r == 0
    assert BM.f_measure([0.5], [0.25], 2.0)[0] == 5.0 * (0.125 / (4 * 0.5 + 0.25))


def test_empty_input_and_negative_bins_are_rejected():
    with pytest.raises(ValueError):
        BM.BinaryMetrics(np.zeros(0), np.zeros(0))
    with pytest.raises(ValueError):
        BM.BinaryMetrics([0.1], [1], num_bins=-1)


# ---- mutants ---------------------------------------------------------------------------------------------
_KEY, _BINS = BM.descending_key, BM.bin_counts                             # the rules the mutants start from


def _ascending_key(scores):
    return ~_KEY(scores)


def _signless_key(scores):
    s = np.asarray(scores, np.float64)
    return _KEY(np.where(s == 0, 0.0, s))


def _lazy_nan_key(scores):
    """NaN handled as numpy's sort would: after every number, and one key per bit pattern."""
    s = np.asarray(scores, np.float64)
    k = _KEY(s)
    return np.where(np.isnan(s), ~np.uint64(0) - (s.view(np.uint64) & np.uint64(0xFF)), k)


def _unmerged_groups(scores, labels):
    key = BM.descending_key(scores)
    order = np.argsort(key, kind="stable")
    pos = BM.is_positive(labels)[order].astype(np.int64)
    return BM.key_score(key[order]), pos, 1 - pos


def _bins_from_last(thresholds, pos, neg, num_bins):
    m = len(thresholds)
    g = m // num_bins if num_bins > 0 else 0
    if g < 2:
        return _BINS(thresholds, pos, neg, num_bins)
    starts = np.arange(0, m, g)
    ends = np.minimum(starts + g, m) - 1
    return np.asarray(thresholds)[ends], np.add.reduceat(pos, starts), np.add.reduceat(neg, starts)


def _pr_from_one(rec, prec):
    return np.concatenate([[[0.0, 1.0]], np.stack([rec, prec], 1)])


MUTANTS = {
    "ascending sort": ("descending_key", _ascending_key),
    "first PR point (0, 1)": ("pr_points", _pr_from_one),
    "ties not merged": ("group_scores", _unmerged_groups),
    "-0.0 == 0.0": ("descending_key", _signless_key),
    "lazy NaN": ("descending_key", _lazy_nan_key),
    "binning from the last score": ("bin_counts", _bins_from_last),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_known_answers_catch_mutant(name, monkeypatch):
    attr, fn = MUTANTS[name]
    monkeypatch.setattr(BM, attr, fn)
    assert known_answer_failures(), name


# ---- independent identity ----------------------------------------------------------------------------------
def mann_whitney(scores, labels):
    """(#[s_p > s_n] + 1/2 #[s_p == s_n]) / (P N), comparing in Spark's key order."""
    k = BM.descending_key(scores)
    pos = BM.is_positive(labels)
    kp, kn = k[pos][:, None], k[~pos][None, :]
    return (float((kp < kn).sum()) + 0.5 * float((kp == kn).sum())) / (kp.size * kn.size)


@pytest.mark.parametrize("seed", range(8))
def test_roc_area_is_the_mann_whitney_statistic(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 3000))
    levels = np.array([math.nan, NAN2, 0.0, -0.0, math.inf, -math.inf, 1e-300, 0.25, 0.5, 0.75, 1.0])
    levels = np.concatenate([levels, rng.random(int(rng.integers(1, 40)))])
    s = levels[rng.integers(0, levels.size, n)]
    y = rng.choice(np.array([0.0, 1.0, 0.3, 0.7, math.nan]), n)
    y[0], y[1] = 1.0, 0.0                                                     # P, N > 0
    m = BM.BinaryMetrics(s, y)
    assert abs(m.area_under_roc() - mann_whitney(s, y)) <= 1e-15
    assert m.positives == int(BM.is_positive(y).sum()) and m.n == n


# ---- binning -----------------------------------------------------------------------------------------------
def literal_bins(thr, pos, neg, num_bins):
    """Spark's counts.mapPartitions(_.grouped(grouping).map(first score, summed counts)) as a plain loop."""
    grouping = len(thr) // num_bins if num_bins else 0
    if grouping < 2:
        return list(thr), list(pos), list(neg)
    out_t, out_p, out_n = [], [], []
    for i in range(0, len(thr), grouping):
        out_t.append(thr[i])
        out_p.append(sum(pos[i:i + grouping]))
        out_n.append(sum(neg[i:i + grouping]))
    return out_t, out_p, out_n


@pytest.mark.parametrize("distinct,num_bins", [(12, 12), (12, 6), (12, 4), (13, 4), (14, 3), (100, 7), (5, 1),
                                               (7, 100)])
def test_binning_matches_the_literal_loop(distinct, num_bins):
    rng = np.random.default_rng(distinct * 101 + num_bins)
    vals = rng.permutation(distinct) / distinct
    s = np.repeat(vals, rng.integers(1, 4, distinct))
    y = rng.integers(0, 2, s.size).astype(np.float64)
    thr, pos, neg = BM.group_scores(s, y)
    want = literal_bins(list(thr), list(pos), list(neg), num_bins)
    m = BM.BinaryMetrics(s, y, num_bins)
    assert m.thresholds().tolist() == want[0]
    assert m.tp.tolist() == np.cumsum(want[1]).tolist() and m.fp.tolist() == np.cumsum(want[2]).tolist()
    g = distinct // num_bins
    if g >= 2 and distinct % g:
        assert len(want[0]) == distinct // g + 1                              # the last run is shorter


# ---- the known answer of neuralcf/002 ------------------------------------------------------------------------
def test_golden_reproduces_from_the_testset():
    import importlib.util
    spec = importlib.util.spec_from_file_location("mk", os.path.join(GOLDEN, "make_binary_metrics_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    p, y = mk.testset_probabilities()
    with open(os.path.join(GOLDEN, "binary_metrics.json")) as f:
        ref = json.load(f)
    m = BM.BinaryMetrics(p.astype(np.float64), y)
    assert (m.n, m.positives, m.negatives, m.thresholds().shape[0]) == \
        (ref["rows"], ref["positives"], ref["negatives"], ref["thresholds"]) == (22440, 12584, 9856, 22419)
    assert m.area_under_roc() == ref["area_under_roc"] and m.area_under_pr() == ref["area_under_pr"]
    for name, arr in (("roc", m.roc()), ("pr", m.pr()), ("threshold_values", m.thresholds()), ("tp", m.tp),
                      ("fp", m.fp)):
        assert arr[ref[name]["index"]].tolist() == ref[name]["values"], name
    with open(os.path.join(GOLDEN, "neuralcf_002_eval.json")) as f:
        ev = json.load(f)
    assert abs(ref["area_under_roc"] - ev["exact_rank_roc_auc"]) <= 1e-14
    assert (ref["keras_roc_auc"], ref["keras_pr_auc"]) == (ev["roc_auc"], ev["pr_auc"])


# ---- C ABI rejections (before any device call) -----------------------------------------------------------
def _create(scores, labels, n, off, n_sets, num_bins):
    from sparrowrecsys_b200 import _lib
    h = C.c_void_p()
    ptr = lambda a: None if a is None else a.ctypes.data                   # noqa: E731
    rc = _lib.load().srs_binary_metrics_create_host(ptr(scores), ptr(labels), n, ptr(off), n_sets, num_bins, 0,
                                                    C.byref(h))
    return rc, h.value


@pytest.mark.parametrize("case", ["n0", "n_huge", "null_scores", "bins", "empty_set", "decreasing", "first",
                                  "last", "n_sets0", "sets_without_offsets", "null_out"])
def test_abi_rejects_before_any_device_call(case):
    from sparrowrecsys_b200 import _lib
    lib = _lib.load()
    s, y = np.array([0.1, 0.2, 0.3]), np.array([0.0, 1.0, 1.0])
    args = dict(scores=s, labels=y, n=3, off=None, n_sets=1, num_bins=0)
    args.update({"n0": dict(n=0), "n_huge": dict(n=2 ** 31), "null_scores": dict(scores=None),
                 "bins": dict(num_bins=-1), "empty_set": dict(off=np.array([0, 1, 1, 3], np.int64), n_sets=3),
                 "decreasing": dict(off=np.array([0, 2, 1, 3], np.int64), n_sets=3),
                 "first": dict(off=np.array([1, 3], np.int64), n_sets=1),
                 "last": dict(off=np.array([0, 2], np.int64), n_sets=1),
                 "n_sets0": dict(off=np.array([0], np.int64), n_sets=0),
                 "sets_without_offsets": dict(n_sets=2), "null_out": {}}[case])
    before = lib.srs_launch_count()
    if case == "null_out":
        rc = lib.srs_binary_metrics_create_host(s.ctypes.data, y.ctypes.data, 3, None, 1, 0, 0, None)
    else:
        rc, h = _create(**args)
        assert h is None
    assert rc == _lib.SRS_ERR_INVALID, lib.srs_last_error()
    assert lib.srs_launch_count() == before


def test_abi_rejects_null_handles():
    from sparrowrecsys_b200 import _lib
    lib = _lib.load()
    out = _lib.SrsBinarySummary()
    assert lib.srs_binary_metrics_summary(None, 0, C.byref(out)) == _lib.SRS_ERR_INVALID
    dst = np.full(4, 7.0)
    assert lib.srs_binary_metrics_curve(None, 0, _lib.SRS_BM_ROC, 1.0, dst.ctypes.data) == _lib.SRS_ERR_INVALID
    assert dst.tolist() == [7.0] * 4
    tp = np.zeros(2, np.int64)
    assert lib.srs_binary_metrics_confusion(None, 0, tp.ctypes.data, tp.ctypes.data) == _lib.SRS_ERR_INVALID
    lib.srs_binary_metrics_destroy(None)


def test_summary_struct_matches_the_header():
    import re
    from sparrowrecsys_b200 import _lib
    with open(os.path.join(ROOT, "include", "srs_ctr.h")) as f:
        body = re.search(r"typedef struct srs_binary_summary \{(.*?)\} srs_binary_summary;", f.read(), re.S).group(1)
    fields = []
    for ctype, names in re.findall(r"(int64_t|double)\s+([^;]+);", body):
        fields += [(n.strip(), {"int64_t": C.c_int64, "double": C.c_double}[ctype]) for n in names.split(",")]
    assert fields == list(_lib.SrsBinarySummary._fields_) and C.sizeof(_lib.SrsBinarySummary) == 48


# ---- the Python front end's helpers ------------------------------------------------------------------------
def test_java_double_layout():
    from sparrowrecsys_b200.evaluation import java_double
    cases = {0.7320829875509305: "0.7320829875509305", 1.0: "1.0", 0.0: "0.0", 0.001: "0.001", 1e-4: "1.0E-4",
             2.5e-10: "2.5E-10", 1e7: "1.0E7", 123.0: "123.0", math.nan: "NaN", -3e-9: "-3.0E-9",
             1.2345e12: "1.2345E12", math.inf: "Infinity", 9.999999e6: "9999999.0"}
    for x, want in list(cases.items()) + [(-0.0, "-0.0")]:
        assert java_double(x) == want, x


def test_evaluation_module_defines_each_name_once():
    import ast
    with open(os.path.join(ROOT, "sparrowrecsys_b200", "evaluation.py")) as f:
        body = ast.parse(f.read()).body
    names = [n.name for n in body if isinstance(n, (ast.FunctionDef, ast.ClassDef))]
    assert len(names) == len(set(names)), names


def test_predictions_csv_and_evaluator_arguments(tmp_path):
    from sparrowrecsys_b200.evaluation import BinaryClassificationEvaluator, read_predictions_csv
    p = tmp_path / "pred.csv"
    p.write_text('label,probability,other\n1,"[0.25,0.75]",x\n0,0.125,y\n')
    prob, lab = read_predictions_csv(str(p))
    assert prob.tolist() == [0.75, 0.125] and lab.tolist() == [1.0, 0.0]
    bad = tmp_path / "bad.csv"
    bad.write_text("label,score\n1,0.5\n")
    with pytest.raises(ValueError):
        read_predictions_csv(str(bad))
    with pytest.raises(ValueError):
        BinaryClassificationEvaluator("accuracy")
