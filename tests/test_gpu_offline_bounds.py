"""Every case of tests/test_offline_bounds.py's `BOUNDS` on the device against its oracle, bit for bit (the binary
metrics' areas within 1e-13 of the exactly rounded sum of the oracle's trapezoids), and a repeat run giving the same
bits."""
import ctypes as C
import re

import numpy as np
import pytest

from oracle import als_cext as X
from oracle import als_implicit_cext as XI
from oracle import feature_job as FQ
from oracle import feature_eng as F
from oracle import graphemb as G
from oracle import item2vec_cext as IX
from oracle import lsh as H
from oracle import lsh_join as LJ
from oracle import als_nnls_cext as XN
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import collab
from sparrowrecsys_b200 import embedding as E
from sparrowrecsys_b200 import featureeng as FE
from sparrowrecsys_b200 import featurejob as FJ

from test_offline_bounds import (BOUNDS, data, discretizer_splits, graph_transitions, i2v_oracle_input,
                                 indexer_oracle, indexer_tokens, labels_csr, nnls_singular_oracle, quantiles,
                                 segmented_metrics, set_curves)

pytestmark = pytest.mark.gpu


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.kind == "f" else a


def _same(a, b, what=""):
    """Bit for bit; a NaN matches any NaN (the device's and the host's default NaNs differ in sign)."""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype.itemsize == b.dtype.itemsize, (what, a.shape, b.shape, a.dtype, b.dtype)
    if a.dtype.kind == "f":
        assert np.array_equal(np.isnan(a), np.isnan(b)), what
        a, b = np.where(np.isnan(a), 0, a).astype(a.dtype), np.where(np.isnan(b), 0, b).astype(b.dtype)
    bad = np.flatnonzero(_bits(a).ravel() != _bits(b).ravel())
    assert bad.size == 0, (what, bad[:5])


def _same_all(xs, ys):
    assert len(xs) == len(ys)
    for i, (x, y) in enumerate(zip(xs, ys)):
        if isinstance(x, (list, tuple)):
            _same_all(x, y)
        else:
            _same(x, y, i)


# ---- per job: (device run, oracle) -------------------------------------------------------------------------------
def _i2v_device(d):
    return E.item2vec(d["ratings"], **d["params"])


def _i2v_oracle(d):
    ids, counts, words, offs, code, point, codelen = i2v_oracle_input(d)
    p = d["params"]
    vec = IX.train(words, offs, counts, code, point, codelen, p["vector_size"], p["window_size"], p["num_iterations"],
                   p["num_partitions"], p["seed"])
    return ids.astype(np.int32), vec


def _graph_device(d):
    r, p = d["ratings"], d["params"]
    tr = E.item_transitions(r)
    out = [[tr[k] for k in ("sources", "out", "row_ptr", "targets", "counts", "dist", "probs")]]
    for W, L in d["walks"]:
        out.append(list(E.random_walks(r, W, L, seed=p["seed"])))
    W, L = d["walks"][-1]
    out.append(list(E.graph_embedding(r, num_walks=W, walk_length=L, **p)))
    return out


def _graph_oracle(d):
    r, p = d["ratings"], d["params"]
    tr = graph_transitions(d)
    out = [[tr["sources"].astype(np.int32), tr["out"].astype(np.int32), tr["row_ptr"].astype(np.int32),
            tr["targets"].astype(np.int32), tr["counts"].astype(np.int32), tr["dist"], tr["probs"]]]
    for W, L in d["walks"]:
        out.append(list(G.random_walks(tr, W, L, seed=p["seed"])))
    W, L = d["walks"][-1]
    ids, vec = G.graph_embedding(r["userId"], r["movieId"], np.rint(r["rating"] * 2), r["timestamp"],
                                 p["vector_size"], p["window_size"], p["num_iterations"], p["num_partitions"],
                                 p["seed"], W, L)
    out.append([ids.astype(np.int32), vec])
    return out


def _lsh_device(d):
    model = E.BucketedRandomProjectionLSHModel(d["uv"], d["bl"])
    out = [model.transform(d["x"])]
    for k in d["ks"]:
        for q, (i, dist) in enumerate(model.approx_nearest_neighbors(d["ids"], d["x"], d["keys"], k)):
            out += [i, dist]
    return out


def _lsh_oracle(d):
    out = [H.transform(d["x"], d["uv"], d["bl"])]
    for k in d["ks"]:
        for key in d["keys"]:
            i, dist = H.approx_nearest_neighbors(d["ids"], d["x"], d["uv"], d["bl"], key, k)
            out += [i, dist]
    return out


def _rec_points(d):
    if "grid" in d:
        return [(d["src"][:s], d["ids"][:t], d["dst"][:t], m) for s, t, m in d["grid"]]
    return [(d["src"], d["ids"], d["dst"], m) for m in d["nums"]]


def _rec_device(d):
    return [list(collab.recommend(s, i, t, m)) for s, i, t, m in _rec_points(d)]


def _rec_oracle(d):
    return [list(X.recommend(s, i, t, m)) for s, i, t, m in _rec_points(d)]


def _fit_device(d):
    out = []
    for k in d["ranks"]:
        m = collab.als({"userId": d["u"], "movieId": d["m"], "rating": d["r"]}, rank=k, seed=k, **d["kw"])
        out.append([m.user_ids, m.user_factors, m.item_ids, m.item_factors])
    return out


def _fit_oracle(d):
    return [list(X.fit(d["u"], d["m"], d["r"], rank=k, seed=k, **d["kw"])) for k in d["ranks"]]


def _folds_device(d):
    r = {"userId": d["u"], "movieId": d["m"], "rating": d["r"]}
    got = collab.als_folds(r, d["fold"], d["n_folds"], d["models"], seed=4)
    return [[m.user_ids, m.user_factors, m.item_ids, m.item_factors] for m in got]


def _folds_single_fits(d):
    out = []
    for spec in d["models"]:
        rows = d["fold"] != spec["exclude_fold"]
        m = collab.als({"userId": d["u"][rows], "movieId": d["m"][rows], "rating": d["r"][rows]}, rank=spec["rank"],
                       max_iter=spec["max_iter"], reg_param=spec["reg_param"], seed=4)
        out.append([m.user_ids, m.user_factors, m.item_ids, m.item_factors])
    return out


def _fe_device(d):
    out = FE.build_samples(d["ratings"], d["movies"], device=0)
    return [out[c] for c in F.COLUMNS]


def _fe_oracle(d):
    out = F.build_samples(d["ratings"], d["movies"])
    return [out[c] for c in F.COLUMNS]


def _p(a):
    return a.ctypes.data


def _fj_device(d):
    op = d["op"]
    if op == "quantile":
        return [FJ.approx_quantile(d["values"], d["probs"], d["eps"])]
    if op == "discretizer":
        out = []
        for N in d["buckets"]:
            bz, b = FJ.QuantileDiscretizer(N, d["eps"]).fit_transform(d["values"])
            out += [bz.splits, b]
        return out
    if op == "bucketize":
        return [FJ.Bucketizer(s).transform(v) for s, v in d["runs"]]
    if op == "scaler":
        out = []
        for v, fit in d["fits"]:
            if fit is None:
                m, x = FJ.MinMaxScaler().fit_transform(v)
                out += [x, np.array([m.original_min, m.original_max])]
            else:
                out.append(FJ.MinMaxScalerModel(*fit).transform(v))
        return out
    if op == "ratings":
        r = FJ.rating_features({"movieId": d["movie"], "rating": d["half"] * 0.5})
        return [r[c] for c in ("movieId", "ratingCount", "avgRating", "ratingVar")]
    if op == "indexer":                                # the raw ABI on word hashes: no 2^20 Python strings
        tok, h = indexer_tokens(d), d["hashes"]
        lw, lc = np.zeros(len(h), np.int32), np.zeros(len(h), np.int64)
        _lib.check(_lib.load().srs_string_indexer_host(_p(tok), tok.size, _p(h), len(h), 0, _p(lw), _p(lc)))
        return [lw, lc]
    if op == "multi_hot":
        r = FJ.multi_hot(d["ids"], d["genres"])
        return [np.array(r["labels"]), r["counts"], r["movieId"], r["offsets"], r["indices"]]
    if op == "split":
        return [FJ.sample_split_rows(n, seed, frac, w) for n, seed, frac, w in d["runs"]]
    if op == "ts_split":
        out = []
        for ts, seed, frac, eps in d["runs"]:
            tr, te, split = FJ.sample_split_rows_by_timestamp(ts, seed, frac, eps)
            out.append([tr, te, np.array([split])])
        return out
    raise KeyError(op)


def _fj_oracle(d):
    op = d["op"]
    if op == "quantile":
        return [quantiles(d["values"], d["probs"], d["eps"])]
    if op == "discretizer":
        out = []
        for N in d["buckets"]:
            s = discretizer_splits(d["values"], N, d["eps"])
            out += [s, FQ.bucketize(s, d["values"])]
        return out
    if op == "bucketize":
        return [FQ.bucketize(s, v) for s, v in d["runs"]]
    if op == "scaler":
        out = []
        with np.errstate(over="ignore", invalid="ignore"):
            for v, fit in d["fits"]:
                if fit is None:
                    x, lo, hi = FQ.min_max_scale(v)
                    out += [x, np.array([lo, hi])]
                else:
                    out.append(FQ.min_max_scale(v, *fit)[0])
        return out
    if op == "ratings":
        ids, n, avg, var = FQ.rating_features(d["movie"], d["half"])
        return [ids, n, avg, var]
    if op == "indexer":
        return list(indexer_oracle(d))
    if op == "multi_hot":
        labels, counts, ids, off, idx = FQ.multi_hot(d["ids"], d["genres"])
        return [np.array(labels), np.array(counts, np.int64), ids, off.astype(np.int32), idx]
    if op == "split":
        return [FQ.split_samples(n, seed, frac, w) for n, seed, frac, w in d["runs"]]
    if op == "ts_split":
        out = []
        for ts, seed, frac, eps in d["runs"]:
            tr, te, split = FQ.split_samples_by_timestamp(ts, seed, frac, eps)
            out.append([tr.astype(np.int64), te.astype(np.int64), np.array([split])])
        return out
    raise KeyError(op)


def _implicit_device(d):
    r = {"userId": d["u"], "movieId": d["m"], "rating": d["r"]}
    return [list(_fit_tuple(collab.als(r, implicit_prefs=True, **f))) for f in d["fits"]]


def _fit_tuple(m):
    return m.user_ids, m.user_factors, m.item_ids, m.item_factors


def _implicit_oracle(d):
    return [list(XI.fit(d["u"], d["m"], d["r"], **f)) for f in d["fits"]]


def _ranking_device(d):
    out = []
    for pred, labels, ks, *_ in d["runs"]:
        off, lab = labels_csr(labels)
        n, L = pred.shape
        for k in ks:
            per, means = np.zeros((3, n)), np.zeros(3)
            _lib.check(_lib.load().srs_ranking_metrics_host(_p(pred), n, L, _p(off), _p(lab if lab.size else off),
                                                            k, 0, _p(per), _p(means)))
            out += [means, per]
    return out


def _ranking_oracle(d):
    out = []
    for pred, labels, ks, *_ in d["runs"]:
        off, lab = labels_csr(labels)
        for k in ks:
            means, per = XI.ranking_metrics(pred, off, lab, k)
            out += [means, per]
    return out


AREA_TOL = 1e-13


def _bm_summaries(m, S):
    """Every set's n, positives, thresholds and both areas (one summary call per set, the struct reused)."""
    f, h = m._lib.srs_binary_metrics_summary, m._h
    out = _lib.SrsBinarySummary()
    ref = C.byref(out)
    n, P, T = np.empty(S, np.int64), np.empty(S, np.int64), np.empty(S, np.int64)
    roc, pr = np.empty(S), np.empty(S)
    for k in range(S):
        _lib.check(f(h, k, ref))
        n[k], P[k], T[k], roc[k], pr[k] = out.n, out.positives, out.thresholds, out.area_under_roc, out.area_under_pr
    return [n, P, T, roc, pr]


def _bm_device(d):
    from sparrowrecsys_b200.evaluation import BinaryClassificationMetrics
    out = []
    for run in d["runs"]:
        s, y, off = run["scores"], run["labels"], run["offsets"]
        if run["path"] == "device":
            import torch
            s, y = torch.from_numpy(s).cuda(), torch.from_numpy(y).cuda()
        with BinaryClassificationMetrics(s, y, 0, off) as m:
            summaries = _bm_summaries(m, len(off) - 1)
            assert summaries[2].min() >= 1                    # every set has a threshold; only then read curves
            curves = [[m.thresholds(k), *m.confusions(k), m.roc(k), m.pr(k), m.precision_by_threshold(k),
                       m.recall_by_threshold(k), m.f_measure_by_threshold(1.0, k)] for k in run["sample"]]
            out.append([summaries, curves])
    return out


def _bm_oracle(d):
    out = []
    for run in d["runs"]:
        R = segmented_metrics(run["scores"].astype(np.float64), run["labels"].astype(np.float64), run["offsets"])
        out.append([[R["n"], R["positives"], np.diff(R["pt_off"]), R["area_roc"], R["area_pr"]],
                    [set_curves(R, k) for k in run["sample"]]])
    return out


def _bm_same(got, want):
    """Counts and curves bit for bit, each area within AREA_TOL."""
    assert len(got) == len(want)
    for (gs, gc), (ws, wc) in zip(got, want):
        _same_all(gs[:3], ws[:3])
        for g, w, what in ((gs[3], ws[3], "roc"), (gs[4], ws[4], "pr")):
            err = np.abs(g - w)
            assert err.max() <= AREA_TOL, (what, int(err.argmax()), err.max())
        _same_all(gc, wc)


def _join_device(d):
    out = []
    for run in d["runs"]:
        model = E.BucketedRandomProjectionLSHModel(run["uv"], run["bl"])
        out.append(list(model.approx_similarity_join(run["ids_a"], run["xa"], run["ids_b"], run["xb"],
                                                     run["threshold"])))
    return out


def _join_oracle(d):
    return [list(LJ.approx_similarity_join(run["ids_a"], run["xa"], run["ids_b"], run["xb"], run["uv"], run["bl"],
                                           run["threshold"])) for run in d["runs"]]


def _nnls_fits_device(d):
    r = {"userId": d["u"], "movieId": d["m"], "rating": d["r"]}
    return [list(_fit_tuple(collab.als(r, nonnegative=True, **f))) for f in d["fits"]]


def _nnls_fits_oracle(d):
    return [list(XN.fit(d["u"], d["m"], d["r"], **f)) for f in d["fits"]]


def _nnls_batch_device(d):
    r = {"userId": d["u"], "movieId": d["m"], "rating": d["r"]}
    return [list(_fit_tuple(m)) for m in collab.als_folds(r, d["fold"], d["n_folds"], d["models"], seed=d["seed"])]


def _nnls_batch_oracle(d):
    """One C-oracle single fit per model on the rows outside its excluded fold: NNLS or Cholesky by its flag."""
    out = []
    for s in d["models"]:
        rows = d["fold"] != s["exclude_fold"]
        fit = XN.fit if s["nonnegative"] else X.fit
        out.append(list(fit(d["u"][rows], d["m"][rows], d["r"][rows], rank=s["rank"], max_iter=s["max_iter"],
                            reg_param=s["reg_param"], seed=d["seed"])))
    return out


def _nnls_singular_device(d):
    out = []
    r = {"userId": d["u"], "movieId": d["m"], "rating": d["r"]}
    for models in d["orders"]:
        try:
            collab.als_folds(r, d["fold"], d["n_folds"], models, seed=d["seed"])
            out.append("no error")
        except ValueError as e:
            hit = re.search(r"model \d+: singular normal equations for \w+ -?\d+ in iteration \d+", str(e))
            out.append(hit.group(0) if hit else str(e))
    return out


def _nnls_device(d):
    if "orders" in d:
        return _nnls_singular_device(d)
    return _nnls_batch_device(d) if "models" in d else _nnls_fits_device(d)


def _nnls_oracle(d):
    if "orders" in d:
        return nnls_singular_oracle(d)
    return _nnls_batch_oracle(d) if "models" in d else _nnls_fits_oracle(d)


def _same_messages(got, want):
    assert got == want


RUNS = {"item2vec": (_i2v_device, _i2v_oracle), "graph": (_graph_device, _graph_oracle),
        "lsh": (_lsh_device, _lsh_oracle), "featureeng": (_fe_device, _fe_oracle),
        "featurejob": (_fj_device, _fj_oracle), "als_implicit": (_implicit_device, _implicit_oracle),
        "ranking_metrics": (_ranking_device, _ranking_oracle), "binary_metrics": (_bm_device, _bm_oracle),
        "lsh_join": (_join_device, _join_oracle), "als_nonnegative": (_nnls_device, _nnls_oracle)}


def _runs(name):
    if name == "als_fit_64_models":
        return _folds_device, _folds_single_fits
    if name.startswith("als_fit"):
        return _fit_device, _fit_oracle
    if name.startswith("als_recommend"):
        return _rec_device, _rec_oracle
    return RUNS[BOUNDS[name].job]


def _compare(name):
    """How a case's device output is held to its oracle's."""
    job = BOUNDS[name].job
    if job == "binary_metrics":
        return _bm_same
    if name == "als_nonnegative_singular_after_nnls":
        return _same_messages
    return _same_all


@pytest.mark.parametrize("name", sorted(BOUNDS))
def test_case_bit_equal_to_its_oracle_and_repeatable(name):
    d = data(name)
    device, oracle = _runs(name)
    got = device(d)
    _compare(name)(got, oracle(d))
    if name == "als_nonnegative_singular_after_nnls":
        assert device(d) == got
    else:
        _same_all(device(d), got)
