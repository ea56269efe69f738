"""Every case of tests/test_offline_bounds.py's `BOUNDS` on the device against its oracle, bit for bit, and a repeat
run giving the same bits."""
import numpy as np
import pytest

from oracle import als_cext as X
from oracle import feature_eng as F
from oracle import graphemb as G
from oracle import item2vec_cext as IX
from oracle import lsh as H
from sparrowrecsys_b200 import collab
from sparrowrecsys_b200 import embedding as E
from sparrowrecsys_b200 import featureeng as FE

from test_offline_bounds import BOUNDS, data, graph_transitions, i2v_oracle_input

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


RUNS = {"item2vec": (_i2v_device, _i2v_oracle), "graph": (_graph_device, _graph_oracle),
        "lsh": (_lsh_device, _lsh_oracle), "featureeng": (_fe_device, _fe_oracle)}


def _runs(name):
    if name == "als_fit_64_models":
        return _folds_device, _folds_single_fits
    if name.startswith("als_fit"):
        return _fit_device, _fit_oracle
    if name.startswith("als_recommend"):
        return _rec_device, _rec_oracle
    return RUNS[BOUNDS[name].job]


@pytest.mark.parametrize("name", sorted(BOUNDS))
def test_case_bit_equal_to_its_oracle_and_repeatable(name):
    d = data(name)
    device, oracle = _runs(name)
    got = device(d)
    _same_all(got, oracle(d))
    _same_all(device(d), got)
