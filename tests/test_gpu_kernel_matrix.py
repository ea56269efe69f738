"""Every kernel instantiation and width regime against the float64 oracle.

The forward kernels are templates over the padded embedding width EP in {12, 16, 32, 64} (`round_ep` in
csrc/model.cu; NCF also over the padded hidden width HP in {16, 32}), and every builder zero-pads the hidden
widths up to a fixed tile.  The defects such code invites - a padded column read as data, the last real
column or unit dropped, the wrong template chosen - only show at a partial pad or at a width limit.  `MATRIX`
names one case per (kernel, EP[, HP]) and width regime: the smallest E of a bucket, a partial pad, the exact
bucket width, hidden width 1 and hidden width at the builder's limit; batch sizes straddle each kernel's row
tile (64 rows: embmlp, embmlp_tc, deepfm2; 32 rows: deepfm, deepfm_tc, din, din_wg, dien; 128-thread CTAs:
ncf).

* GPU: each case asserts its kernel, matches the float64 oracle and repeats bit for bit.
* CPU: the tolerances of the GPU test see, at every case, the column E - 1 of the embedding tables zeroed and
  the last real unit of each hidden layer zeroed; and `MATRIX` reaches every instantiation the launchers in
  csrc/*.cu dispatch, so a new instantiation without a parity case fails here.
"""
import collections
import glob
import os
import re
import zlib

import numpy as np
import pytest

from oracle import ctr_oracle as O
from sparrowrecsys_b200.features import synthetic_features
from sparrowrecsys_b200.spec import default_spec, history_keys
from sparrowrecsys_b200.weights import init_weights

PROB_ATOL = 2e-5
LOGIT_ATOL = 2e-4
WIDE_LOGIT_ATOL = 5e-4          # DIEN, and DIN at E > 32 (as in test_seq_dien.py / test_gpu_parity.py)
N_MOVIES, N_USERS = 1000, 1200  # small vocabularies keep the oracle fast
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc")

# rows per CTA tile of each kernel; a case's batch is one tile + 1
ROWS = {"ncf_kernel": 257, "embmlp_kernel": 129, "embmlp_tc_kernel": 129, "deepfm2_kernel": 129,
        "deepfm_kernel": 65, "deepfm_tc_kernel": 65, "din_kernel": 65, "din_wg_kernel": 65, "dien_kernel": 65}
IMPL_OPTION = {"embeddingmlp": "embmlp_impl", "widendeep": "embmlp_impl", "deepfm": "deepfm_impl",
               "din": "din_impl"}

Case = collections.namedtuple("Case", "model over impl B kernel")


def _case(model, kernel, impl=None, **over):
    return Case(model, over, impl, ROWS[kernel.split("<")[0]], kernel)


NCF, TT = "ncf_kernel<neural_cf_model_1>", "ncf_kernel<two_towers>"
EMB, EMB_WD = "embmlp_kernel", "embmlp_kernel<wide&deep>"
EMB_TC, EMB_TC_WD = "embmlp_tc_kernel", "embmlp_tc_kernel<wide&deep>"

MATRIX = [
    # ---- ncf_kernel<EP, HP>: every (EP, HP) pair, hidden 1 / 16 / 17 / 32 and three layers ----
    _case("neuralcf", NCF, emb_dim=1, hidden=(1,)),
    _case("neuralcf", NCF, emb_dim=12, hidden=(17, 9)),
    _case("neuralcf", NCF, emb_dim=13, hidden=(16, 16)),
    _case("neuralcf", NCF, emb_dim=16, hidden=(32, 32, 32)),
    _case("neuralcf", NCF, emb_dim=17, hidden=(1,)),
    _case("neuralcf", NCF, emb_dim=32, hidden=(17, 9)),
    _case("neuralcf", NCF, emb_dim=33, hidden=(16, 16)),
    _case("neuralcf", NCF, emb_dim=64, hidden=(32, 32, 32)),
    _case("twotowers", TT, emb_dim=13, hidden=(17, 9), final_dense=True),
    _case("twotowers", TT, emb_dim=16, hidden=(1,), final_dense=False),
    _case("twotowers", TT, emb_dim=17, hidden=(16, 16), final_dense=False),
    _case("twotowers", TT, emb_dim=32, hidden=(32, 32, 32), final_dense=True),
    _case("twotowers", TT, emb_dim=33, hidden=(1,), final_dense=True),
    _case("twotowers", TT, emb_dim=64, hidden=(17, 9), final_dense=False),
    _case("twotowers", TT, emb_dim=64, hidden=(16, 16), final_dense=True),
    # ---- embmlp_kernel<EP> (CUDA cores; the default above E = 12) and embmlp_tc_kernel (E <= 12) ----
    _case("embeddingmlp", EMB, emb_dim=13),
    _case("widendeep", EMB_WD, emb_dim=17),
    _case("embeddingmlp", EMB, emb_dim=31),
    _case("widendeep", EMB_WD, emb_dim=33),
    _case("embeddingmlp", EMB, emb_dim=64),
    _case("widendeep", EMB_TC_WD, emb_dim=1),
    _case("embeddingmlp", EMB_TC, emb_dim=10, hidden=(1, 1)),
    _case("widendeep", EMB_TC_WD, emb_dim=10, hidden=(127, 128)),
    _case("embeddingmlp", EMB_TC, emb_dim=10, hidden=(128, 1)),
    _case("widendeep", EMB_WD, "cudacore", emb_dim=10, hidden=(1, 1)),
    _case("embeddingmlp", EMB, "cudacore", emb_dim=10, hidden=(127, 128)),
    _case("widendeep", EMB_WD, "cudacore", emb_dim=10, hidden=(128, 1)),
    _case("embeddingmlp", EMB, emb_dim=64, hidden=(1, 1)),
    _case("widendeep", EMB_WD, emb_dim=64, hidden=(127, 128)),
    _case("embeddingmlp", EMB, emb_dim=64, hidden=(128, 1)),
    # W&D wide part: one bucket, a prime count, 2^20
    _case("widendeep", EMB_TC_WD, emb_dim=10, cross_buckets=1),
    _case("widendeep", EMB_WD, emb_dim=17, cross_buckets=97),
    _case("widendeep", EMB_TC_WD, emb_dim=10, cross_buckets=1 << 20),
    # ---- deepfm_tc_kernel (12 < E <= 16) and deepfm_kernel<EP> ----
    _case("deepfm", "deepfm_tc_kernel", emb_dim=13),
    _case("deepfm", "deepfm_tc_kernel", emb_dim=15),
    _case("deepfm", "deepfm_kernel", emb_dim=12, hidden=(17, 33)),
    _case("deepfm", "deepfm_kernel", "cudacore", emb_dim=13),
    _case("deepfm", "deepfm_kernel", emb_dim=17),
    _case("deepfm", "deepfm_kernel", emb_dim=33),
    _case("deepfm", "deepfm_kernel", emb_dim=64),
    *[_case("deepfm", "deepfm_tc_kernel", emb_dim=16, hidden=h) for h in ((1, 1), (63, 64), (64, 1), (17, 33))],
    *[_case("deepfm", "deepfm_kernel", "cudacore", emb_dim=16, hidden=h)
      for h in ((1, 1), (63, 64), (64, 1), (17, 33))],
    *[_case("deepfm", "deepfm_kernel", emb_dim=64, hidden=h) for h in ((1, 1), (63, 64), (64, 1), (17, 33))],
    # ---- deepfm2_kernel<EP> ----
    _case("deepfm_v2", "deepfm2_kernel", emb_dim=10, hidden=(1, 1)),
    _case("deepfm_v2", "deepfm2_kernel", emb_dim=13),
    _case("deepfm_v2", "deepfm2_kernel", emb_dim=15, hidden=(17, 3)),
    _case("deepfm_v2", "deepfm2_kernel", emb_dim=16, hidden=(31, 15)),
    _case("deepfm_v2", "deepfm2_kernel", emb_dim=17, hidden=(1, 1)),
    _case("deepfm_v2", "deepfm2_kernel", emb_dim=33, hidden=(31, 15)),
    _case("deepfm_v2", "deepfm2_kernel", emb_dim=64, hidden=(17, 3)),
    # ---- din_kernel<EP> (the default at T <= 8 or E <= 16) and din_wg_kernel<32|64> (the default above) ----
    _case("din", "din_kernel", emb_dim=12, hist_len=3),
    _case("din", "din_kernel", emb_dim=13, hist_len=12),
    _case("din", "din_kernel", emb_dim=32, hist_len=8),
    _case("din", "din_kernel", emb_dim=64, hist_len=5),
    _case("din", "din_kernel", "cudacore", emb_dim=33, hist_len=12),
    _case("din", "din_kernel", "cudacore", emb_dim=63, hist_len=12),
    *[_case("din", "din_wg_kernel", emb_dim=E, hist_len=12, hidden=h)
      for E in (32, 64) for h in ((1, 1), (65, 33), (128, 1))],
    # ---- dien_kernel<EP> ----
    _case("dien", "dien_kernel", emb_dim=12, hist_len=6, hidden=(1, 1)),
    _case("dien", "dien_kernel", emb_dim=13, hist_len=6),
    _case("dien", "dien_kernel", emb_dim=15, hist_len=6, hidden=(65, 33)),
    _case("dien", "dien_kernel", emb_dim=31, hist_len=6),
    _case("dien", "dien_kernel", emb_dim=31, hist_len=6, hidden=(1, 1)),
    _case("dien", "dien_kernel", emb_dim=32, hist_len=6, hidden=(65, 33)),
]


def _case_id(c):
    parts = [c.model, "E%d" % c.over["emb_dim"]]
    for k, v in sorted(c.over.items()):
        if k == "hidden":
            parts.append("h" + "x".join(map(str, v)))
        elif k == "hist_len":
            parts.append("T%d" % v)
        elif k == "cross_buckets":
            parts.append("cb%d" % v)
        elif k == "final_dense":
            parts.append("fd" if v else "dot")
    parts.append(c.impl or "default")
    return "-".join(parts)


def _spec(c):
    return default_spec(c.model, n_movies=N_MOVIES, n_users=N_USERS, **c.over)


def _seed(c):
    return zlib.crc32(_case_id(c).encode()) & 0xFFFF


def _output_rows(spec):
    """The output Dense's kernel rows that the embeddings and hidden layers feed (not the one-hot weights)."""
    h = spec.hidden
    if spec.model in ("embeddingmlp", "widendeep"):
        return "dense_2/kernel", slice(0, h[-1])
    if spec.model == "deepfm":
        return "dense_2/kernel", slice(spec.fm1_width, None)             # the 4 FM dots and the deep part
    if spec.model == "deepfm_v2":
        return "out/kernel", slice(1, None)                              # the FM term and the deep part
    if spec.model == "neuralcf":
        return "dense_%d/kernel" % len(h), slice(None)
    if spec.model == "twotowers":
        return ("dense_out/kernel", slice(None)) if spec.final_dense else (None, None)
    return "dense_2/kernel", slice(None)


def _weights(c):
    """Reference initialisers, stressed so that a lost embedding column or hidden unit shows in the logit:
    * every embedding table x3 (DIN's and DIEN's behaviour table, +-0.05 under the reference initialiser, x10;
      DIEN's attention unit x4, as `_stress_weights` in test_seq_dien.py);
    * the output Dense's rows fed by the network x4 (x10 for DeepFM, whose glorot limit is set by the ~2000
      one-hot rows beside them), the last hidden unit's weight at least 0.25 in magnitude;
    * DeepFM_v2 keeps its scale (its FM term is quadratic in the projections and already moves the logit);
    * the last unit of each ReLU hidden layer biased to |b| + 0.5, so that it is live on the batch."""
    spec = _spec(c)
    W = init_weights(spec, _seed(c))
    for k in _embedding_tables(W):
        W[k] = W[k] * np.float32(10.0 if k == "embedding" else 1.0 if spec.model == "deepfm_v2" else 3.0)
    if spec.model == "dien":
        for k in ("att_dense/kernel", "att_out/kernel"):
            W[k] = W[k] * np.float32(4.0)
    name, rows = _output_rows(spec)
    if name:
        W[name] = W[name].copy()
        W[name][rows] *= np.float32({"deepfm": 10.0, "deepfm_v2": 1.0}.get(spec.model, 4.0))
        last = (rows.stop or W[name].shape[0]) - 1                       # the last hidden unit's weight
        W[name][last] = np.copysign(max(abs(W[name][last, 0]), 0.25), W[name][last])
    if spec.model not in ("din", "dien"):                                # PReLU layers are never dead
        for layer in _hidden_layers(spec):
            W[layer + "/bias"] = W[layer + "/bias"].copy()
            W[layer + "/bias"][-1] = abs(W[layer + "/bias"][-1]) + np.float32(0.5)
    return W


def _features(c):
    """Zipf ids with 10 % missing genres, plus the ends of both vocabularies in the first rows."""
    spec = _spec(c)
    f = synthetic_features(spec, c.B, seed=_seed(c))
    f["movieId"][:4] = [0, N_MOVIES - 1, N_MOVIES - 1, 0]
    f["userId"][:4] = [N_USERS - 1, 0, N_USERS - 1, 0]
    keys = history_keys(spec.hist_len) if c.model in ("din", "dien") else ["userRatedMovie1"]
    for k in keys:
        f[k][1] = N_MOVIES - 1
    f[keys[0]][2] = 0
    f[keys[-1]][3] = N_MOVIES - 1
    return f


def _logit_atol(c):
    if c.model == "dien" or (c.model == "din" and c.over["emb_dim"] > 32):
        return WIDE_LOGIT_ATOL
    return LOGIT_ATOL


def _model(c, W):
    from sparrowrecsys_b200.model import CTRModel
    return CTRModel(_spec(c), W, device=0, options={IMPL_OPTION[c.model]: c.impl} if c.impl else None)


def round_ep(E):
    """csrc/model.cu round_ep: the padded embedding width every templated kernel is instantiated over."""
    return 12 if E <= 12 else 16 if E <= 16 else 32 if E <= 32 else 64


def instantiation(c):
    """(kernel, EP[, HP]) a case runs; the tensor-core EmbeddingMLP / DeepFM kernels are not templates."""
    base = c.kernel.split("<")[0]
    spec = _spec(c)
    if base in ("embmlp_tc_kernel", "deepfm_tc_kernel"):
        return (base,)
    if base == "ncf_kernel":                          # build_ncf: HP = 16 if max(hidden) <= 16 else 32
        return (base, round_ep(spec.emb_dim), 16 if max(spec.hidden) <= 16 else 32)
    return (base, round_ep(spec.emb_dim))


def dispatched_instantiations():
    """Every (kernel, EP[, HP]) the launchers in csrc/*.cu can dispatch, read from their dispatch lines."""
    found = set()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        with open(path) as f:
            src = f.read()
        for ep, name, ep2 in re.findall(r"case (\d+): return launch_(\w+?)_t<(\d+)>", src):
            assert ep == ep2, (path, ep, name, ep2)
            found.add((name + "_kernel", int(ep)))
        for ep, hp in re.findall(r"SRS_NCF_CASE\((\d+), (\d+)\)", src):
            found.add(("ncf_kernel", int(ep), int(hp)))
        for ep in re.findall(r"din_wg_kernel<(\d+)><<<", src):
            found.add(("din_wg_kernel", int(ep)))
    return found


def _embedding_tables(W):
    return [k for k in W if k == "embedding" or k.endswith("_embedding")]


def _hidden_layers(spec):
    n = len(spec.hidden)
    if spec.model == "neuralcf":
        return ["dense_%d" % i for i in range(n)]
    if spec.model == "twotowers":
        return ["%s_dense_%d" % (side, i) for side in ("item", "user") for i in range(n)]
    if spec.model == "deepfm_v2":
        return ["deep", "deep_1"]
    return ["dense", "dense_1"]


def _defect_probes(spec, W):
    """(name, weights) pairs: column E - 1 of every embedding table zeroed, and for each hidden layer its last
    real unit (kernel column h - 1 and bias h - 1) zeroed."""
    E = spec.emb_dim
    Wc = dict(W)
    for k in _embedding_tables(W):
        Wc[k] = W[k].copy()
        Wc[k][:, E - 1] = 0
    yield "embedding column %d" % (E - 1), Wc
    for layer in _hidden_layers(spec):
        Wu = dict(W)
        h = W[layer + "/kernel"].shape[1]
        Wu[layer + "/kernel"] = W[layer + "/kernel"].copy()
        Wu[layer + "/kernel"][:, h - 1] = 0
        Wu[layer + "/bias"] = W[layer + "/bias"].copy()
        Wu[layer + "/bias"][h - 1] = 0
        yield "%s unit %d" % (layer, h - 1), Wu


# ---- CPU: the table is complete and its tolerances can see the defects ---------------------------------
def test_matrix_reaches_every_dispatched_instantiation():
    dispatched = dispatched_instantiations()
    assert {d[0] for d in dispatched} == {"ncf_kernel", "embmlp_kernel", "deepfm_kernel", "deepfm2_kernel",
                                          "din_kernel", "din_wg_kernel", "dien_kernel"}, dispatched
    reached = {instantiation(c) for c in MATRIX}
    missing = sorted(dispatched - reached)
    assert not missing, "no MATRIX case runs %s" % ", ".join("%s<%s>" % (d[0], ", ".join(map(str, d[1:])))
                                                             for d in missing)


def test_matrix_cases_are_distinct():
    ids = [_case_id(c) for c in MATRIX]
    assert len(ids) == len(set(ids))


@pytest.mark.parametrize("case", MATRIX, ids=_case_id)
def test_tolerance_sees_a_dropped_column_or_unit(case):
    """The oracle with a defect a kernel could have - the last real embedding column or hidden unit lost -
    differs from the intact oracle by more than 10x the logit tolerance the GPU case is held to."""
    spec, W, f = _spec(case), _weights(case), _features(case)
    _, z = O.forward(spec, W, f, dtype=np.float64)
    floor = 10 * _logit_atol(case)
    for name, Wd in _defect_probes(spec, W):
        _, zd = O.forward(spec, Wd, f, dtype=np.float64)
        assert np.abs(zd - z).max() > floor, "%s moves the logit by only %.3g" % (name, np.abs(zd - z).max())


# ---- GPU: every case against the float64 oracle ------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", MATRIX, ids=_case_id)
def test_kernel_matches_float64_oracle(case):
    spec, W, f = _spec(case), _weights(case), _features(case)
    with _model(case, W) as m:
        assert m.kernel_name == case.kernel
        p, z = m.predict_with_logits(f)
        p2, z2 = m.predict_with_logits(f)
    assert np.array_equal(p, p2) and np.array_equal(z, z2)           # a second call gives the same bits
    po, zo = O.forward(spec, W, f, dtype=np.float64)
    assert p.shape == (case.B, 1) and p.dtype == np.float32
    assert np.abs(z - zo).max() <= _logit_atol(case), "logit err %g" % np.abs(z - zo).max()
    assert np.abs(p - po).max() <= PROB_ATOL, "prob err %g" % np.abs(p - po).max()


# one past each builder's width limit: ValueError when the model is created, and nothing is launched
@pytest.mark.gpu
@pytest.mark.parametrize("model,hidden", [
    ("neuralcf", (33,)), ("neuralcf", (16, 33)), ("twotowers", (33,)), ("neuralcf", (8, 8, 8, 8)),
    ("embeddingmlp", (129, 128)), ("widendeep", (128, 129)), ("deepfm", (65, 64)), ("deepfm", (64, 65)),
    ("deepfm_v2", (33, 16)), ("deepfm_v2", (32, 17)), ("din", (129, 64)), ("din", (128, 65)),
    ("dien", (129, 64)), ("dien", (128, 65))])
def test_width_one_past_the_builder_limit_is_rejected(model, hidden):
    from sparrowrecsys_b200.model import CTRModel, launch_count
    spec = default_spec(model, hidden=hidden, n_movies=N_MOVIES, n_users=N_USERS)
    W = init_weights(spec, 0)
    before = launch_count()
    with pytest.raises(ValueError, match="hidden"):
        CTRModel(spec, W, device=0)
    assert launch_count() == before


@pytest.mark.gpu
@pytest.mark.parametrize("model,E,kernel", [("embeddingmlp", 10, EMB_TC), ("widendeep", 10, EMB_TC_WD),
                                            ("deepfm", 16, "deepfm_tc_kernel")])
def test_tensor_core_mlps_at_trained_magnitudes(model, E, kernel):
    """Trained-scale weights (embeddings x10, the output Dense x4, as DIN's test_top_mlp_trained_magnitudes):
    the bf16x3 split must hold the north-star 1e-4 on probabilities where one bf16 product would not."""
    from sparrowrecsys_b200.model import CTRModel
    spec = default_spec(model, emb_dim=E, n_movies=N_MOVIES, n_users=N_USERS)
    W = init_weights(spec, 23)
    for k in _embedding_tables(W):
        W[k] = (W[k] * 10).astype(np.float32)
    W["dense_2/kernel"] = (W["dense_2/kernel"] * 4).astype(np.float32)
    f = synthetic_features(spec, 2048, seed=23)
    with CTRModel(spec, W, device=0) as m:
        assert m.kernel_name == kernel
        p, z = m.predict_with_logits(f)
    po, zo = O.forward(spec, W, f, dtype=np.float64)
    assert np.abs(zo).max() > 2.0
    assert np.abs(p - po).max() <= 1e-4, np.abs(p - po).max()
    assert np.abs(z - zo).max() <= 1e-3 * max(1.0, np.abs(zo).max()), np.abs(z - zo).max()


@pytest.mark.gpu
@pytest.mark.parametrize("model,E,kernel", [("widendeep", 10, EMB_TC_WD), ("deepfm", 16, "deepfm_tc_kernel")])
@pytest.mark.parametrize("n_streams", [1, 2])
def test_back_to_back_tensor_core_launches_match_serial(model, E, kernel, n_streams):
    """Both kernels are launched with programmatic dependent launch (griddepcontrol): eight launches alternating
    two batches, queued without a host sync on one stream or on two (each capped to half the SMs, as bench.py
    runs), give the bits of the serial calls."""
    import torch
    from sparrowrecsys_b200.model import CTRModel
    spec = default_spec(model, emb_dim=E, n_movies=N_MOVIES, n_users=N_USERS)
    W = init_weights(spec, 29)
    fa, fb = synthetic_features(spec, 3001, seed=1), synthetic_features(spec, 4099, seed=2)
    with CTRModel(spec, W, device=0) as m:
        assert m.kernel_name == kernel
        ra, rb = m.predict(fa)[:, 0], m.predict(fb)[:, 0]
        da, db = m.to_device(fa), m.to_device(fb)
        if n_streams == 2:
            m.set_sm_limit(torch.cuda.get_device_properties(0).multi_processor_count // 2)
        streams = [torch.cuda.Stream() for _ in range(n_streams)]
        batches = [da if i % 2 == 0 else db for i in range(8)]
        outs = [torch.empty(d.B, dtype=torch.float32, device="cuda:0") for d in batches]
        for s in streams:
            s.wait_stream(torch.cuda.current_stream())
        for i, d in enumerate(batches):
            m.predict_device(d, outs[i], stream=streams[i % n_streams])
        for s in streams:
            torch.cuda.current_stream().wait_stream(s)
        m.status()
        for i, out in enumerate(outs):
            assert np.array_equal(out.cpu().numpy(), ra if i % 2 == 0 else rb), i
