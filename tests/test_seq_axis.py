"""The history axis of the sequence kernels against the float64 oracle: `SEQ_MATRIX` and its CPU checks.

DIN and DIEN are the only models with a history, and their kernels walk it in ways the other axes never reach:
* `din_kernel<EP>` (csrc/din.cu) stages `kDinChunk` positions per warp at a time and reads the PReLU alpha of
  position t0 + t; a partial chunk after a full one, or an alpha taken from the wrong chunk, shows only at
  T = c - 1, c, c + 1, 2c, 2c + 1;
* `dien_kernel<EP, AUX>` (csrc/dien.cu) walks the history one step at a time with no bound on T; the step kernel
  of `fit` trains up to `kDienMaxT` positions (csrc/kernels.h), so its T edges are 63, 64 and 65, and 200 is the
  long-history shape of BASELINE;
* every sequence kernel passes movie ids through float32 (DIN.py:95,125, DIEN.py:96-105): above 2^24 an id reads
  the row of its rounding (2^24 + 1 -> 2^24, 2^24 + 3 -> 2^24 + 4), which only a vocabulary past 2^24 shows.

Each case names its kernel, E, T, batch and vocabulary.  Its batch holds the history patterns where kernels go
wrong (`features`): an all-padding row, padding only at position 0 and only at T - 1, padding on both sides of each
chunk boundary, a candidate that is also in its own history; a case past 2^24 also holds the ids around 2^24.  The
behaviour table is x10 the reference initialiser and its row 0 is stressed, because DIN pools padding as row 0
while DIEN masks it.

* CPU (this file): every dispatched instantiation has a case at T = c - 1, c and c + 1 of its chunk and every
  sequence kernel a case past 2^24; each case's inputs reach the edges it stands for; and each defect a kernel
  could have moves some row's logit (or aux) past the tolerance of every case's GPU check, and past 10x that
  tolerance in some case of each kernel.
* GPU (tests/test_gpu_seq_axis.py): each case runs its kernel, matches the float64 oracle and repeats bit for bit.
"""
import collections
import functools
import os
import re
import zlib

import numpy as np
import pytest

from oracle import ctr_oracle as O
from sparrowrecsys_b200.features import negative_history_keys, synthetic_features
from sparrowrecsys_b200.spec import default_spec, history_keys
from sparrowrecsys_b200.weights import init_aux_weights, init_weights

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sparrowrecsys_b200", "csrc")

PROB_ATOL = 2e-5
LOGIT_ATOL = 2e-4
WIDE_LOGIT_ATOL = 5e-4          # DIEN, and DIN at E > 32 (as in test_gpu_kernel_matrix.py)
AUX_RTOL, AUX_ATOL = 1e-5, 1e-6  # aux[B] (as test_dien_aux.py)
SMALL_VOCAB, N_USERS = 1000, 1200
TWO24 = 1 << 24
BIG_VOCAB = TWO24 + 4           # 2^24 + 3 is in range raw and rounds to 2^24 + 4: out of range
ROUNDS_DOWN, EXACT, ROUNDS_OUT = TWO24 + 1, TWO24 + 2, TWO24 + 3
TABLE_SCALE = np.float32(10.0)  # the behaviour table is x10 the reference's +-0.05
TABLE_SEED, TABLE_LO, TABLE_HI = 4242, -0.5, 0.5   # srs_fill_uniform's draw of the tables past 2^24


def source_constant(fname, name, src_dir=CSRC):
    with open(os.path.join(src_dir, fname)) as f:
        m = re.search(r"constexpr int %s = (\d+);" % name, f.read())
    assert m, "%s not found in %s" % (name, fname)
    return int(m.group(1))


DIN_CHUNK = source_constant("din.cu", "kDinChunk")
WG_POS = source_constant("din_wg.cu", "kWgPos")
DIEN_MAX_T = source_constant("kernels.h", "kDienMaxT")

Case = collections.namedtuple("Case", "name model kernel aux impl E T B vocab")


def _case(model, kernel, E, T, B, vocab=SMALL_VOCAB, aux=False, impl=None):
    tag = {"din_kernel": "din", "din_wg_kernel": "din_wg", "dien_kernel": "dien_aux" if aux else "dien",
           "dien_train_step_kernel": "dien_fit"}[kernel]
    name = "%s-E%d-T%d-B%d%s" % (tag, E, T, B, "-past2^24" if vocab > TWO24 else "")
    return Case(name, model, kernel, aux, impl, E, T, B, vocab)


# T values are literal, so that a changed chunk in the source leaves the guard below something to name
SEQ_MATRIX = [
    # ---- din_kernel<EP>: a partial chunk, one full chunk, a full then a partial one, two, two and a partial;
    #      E 32 / 64 force the CUDA-core kernel, which the default replaces with din_wg_kernel above T = 8 ----
    *[_case("din", "din_kernel", E, T, B, impl="cudacore" if E > 16 else None)
      for E in (10, 16, 32, 64) for T, B in ((31, 33), (32, 97), (33, 33), (64, 97), (65, 33))],
    _case("din", "din_kernel", 64, 200, 97, impl="cudacore"),
    # ---- dien_kernel<EP, false> and <EP, true>: one step, two, either side of kDienMaxT, BASELINE's 200 ----
    *[_case("dien", "dien_kernel", E, T, B, aux=aux)
      for aux in (False, True) for E in (10, 16, 32)
      for T, B in ((1, 33), (2, 97), (63, 33), (64, 97), (65, 33), (200, 97))],
    # ---- ids past 2^24 ----
    _case("din", "din_kernel", 10, 33, 33, BIG_VOCAB),
    _case("din", "din_wg_kernel", 32, 65, 33, BIG_VOCAB),
    _case("dien", "dien_kernel", 10, 65, 33, BIG_VOCAB),
    _case("dien", "dien_kernel", 10, 65, 33, BIG_VOCAB, aux=True),
    _case("dien", "dien_train_step_kernel", 10, 64, 33, BIG_VOCAB),
]
FIT_BATCH = 12                  # the fit case trains its rows in steps of 12, 12 and 9


def chunk(case):
    """The positions a kernel takes at a time: its T edges are c - 1, c and c + 1."""
    return {"din_kernel": DIN_CHUNK, "din_wg_kernel": WG_POS}.get(case.kernel, DIEN_MAX_T)


def round_ep(E):
    return 12 if E <= 12 else 16 if E <= 16 else 32 if E <= 32 else 64


def instantiation(case):
    return (case.kernel, round_ep(case.E), case.aux)


def past_2_24(case):
    return case.vocab > TWO24


def dispatched_instantiations(src_dir=CSRC):
    """(kernel, EP, AUX) of every sequence-kernel launch in the dispatch switches of csrc/din.cu, din_wg.cu and
    dien.cu."""
    src = {f: open(os.path.join(src_dir, f)).read() for f in ("din.cu", "din_wg.cu", "dien.cu")}
    found = {("din_kernel", int(ep), False) for ep in re.findall(r"launch_din_t<(\d+)>\(", src["din.cu"])}
    found |= {("din_wg_kernel", int(ep), False) for ep in re.findall(r"din_wg_kernel<(\d+)><<<", src["din_wg.cu"])}
    found |= {("dien_kernel", int(ep), False) for ep in re.findall(r"launch_dien_t<(\d+)>\(", src["dien.cu"])}
    found |= {("dien_kernel", int(ep), True) for ep in re.findall(r"launch_dien_t<(\d+), true>\(", src["dien.cu"])}
    return found


def coverage_gaps(matrix, src_dir=CSRC):
    """What `matrix` lacks, as readable lines: for each dispatched instantiation but din_wg_kernel's (whose chunks
    have their own files), the T values c - 1, c, c + 1 of its chunk without a case; for each sequence kernel, a
    case past 2^24."""
    chunks = {"din_kernel": source_constant("din.cu", "kDinChunk", src_dir),
              "dien_kernel": source_constant("kernels.h", "kDienMaxT", src_dir)}
    gaps = []
    for kernel, ep, aux in sorted(dispatched_instantiations(src_dir)):
        label = "%s<%d%s>" % (kernel, ep, ", true" if aux else "")
        if kernel in chunks:
            c = chunks[kernel]
            have = {case.T for case in matrix if instantiation(case) == (kernel, ep, aux)}
            missing = [T for T in (c - 1, c, c + 1) if T not in have]
            if missing:
                gaps.append("%s: no case at T = %s (chunk %d)" % (label, ", ".join(map(str, missing)), c))
    for kernel, aux in sorted({(k, a) for k, _, a in dispatched_instantiations(src_dir)} |
                              {("dien_train_step_kernel", False)}):
        if not any(past_2_24(c) and (c.kernel, c.aux) == (kernel, aux) for c in matrix):
            gaps.append("%s%s: no case past 2^24" % (kernel, "<AUX>" if aux else ""))
    return gaps


# ---- a case's inputs ----------------------------------------------------------------------------------------
def spec_of(case, vocab=None):
    return default_spec(case.model, emb_dim=case.E, hist_len=case.T, n_movies=vocab or case.vocab, n_users=N_USERS)


def seed_of(case):
    return zlib.crc32(case.name.encode()) & 0xFFFF


def row0(E):
    """The stressed table row 0: |x| in [0.3, 0.5] with alternating signs, far from a zero row."""
    return (np.linspace(0.3, 0.5, E) * np.where(np.arange(E) % 2, -1.0, 1.0)).astype(np.float32)


def weights(case):
    """Reference initialisers with non-zero biases and alphas (init_weights' for_test), the behaviour table x10
    with the stressed row 0, DIEN's attention x4 (as test_seq_dien.py), the auxiliary head for AUX and fit.  Past
    2^24 the behaviour table is left out: it is `big_table_rows`' formula, generated on the device."""
    spec = spec_of(case)
    W = init_weights(spec, seed_of(case), skip=("embedding",) if past_2_24(case) else ())
    if not past_2_24(case):
        W["embedding"] = W["embedding"] * TABLE_SCALE
        W["embedding"][0] = row0(case.E)
    if case.model == "dien":
        for k in ("att_dense/kernel", "att_out/kernel"):
            W[k] = W[k] * np.float32(4.0)
        W["dense/kernel"] = W["dense/kernel"].copy()
        W["dense/kernel"][:case.E] *= np.float32(4.0)                # the rows u_T feeds
    W["dense_2/kernel"] = W["dense_2/kernel"] * np.float32(4.0)
    if case.aux or case.kernel == "dien_train_step_kernel":
        W.update(init_aux_weights(spec, seed_of(case)))
        rng = np.random.default_rng(seed_of(case) + 1)
        for k in W:
            if k.startswith("aux_") and k.endswith("/bias"):
                W[k] = rng.uniform(-0.3, 0.3, size=W[k].shape).astype(np.float32)
    return W


def big_table_rows(rows, E):
    """Rows `rows` of a table past 2^24: srs_fill_uniform(TABLE_SEED, -0.5, 0.5) over [V][E], row 0 stressed."""
    rows = np.asarray(rows, np.int64)
    flat = (rows[:, None] * E + np.arange(E)[None, :]).reshape(-1)
    out = O.fill_uniform(flat, TABLE_SEED, TABLE_LO, TABLE_HI).reshape(-1, E)
    out[rows == 0] = row0(E)
    return out


def history_of(case, f):
    """[B, T] history ids in graph position order, as int64."""
    return np.stack([np.asarray(f[k]).astype(np.int64) for k in history_keys(case.T)], axis=1)


def features(case):
    """The case's batch.  Rows 0-4 carry the history patterns, rows 5-9 past 2^24 the ids around 2^24, the rest
    draw a random length and pad the tail as the reference's samples do.
      row 0  all padding               row 3  padding at c - 1 and c of every chunk boundary c < T
      row 1  padding only at 0         row 4  its candidate at position T // 2 and T - 1 of its history
      row 2  padding only at T - 1
    Negatives (DIEN) and labels are drawn for every case."""
    spec = spec_of(case)
    T, B, c = case.T, case.B, chunk(case)
    rng = np.random.default_rng(seed_of(case))
    f = synthetic_features(spec, B, seed=seed_of(case))
    top = min(case.vocab, 5000)
    H = rng.integers(1, top, size=(B, T))
    lens = rng.integers(1, T + 1, size=B)
    tail = np.arange(T)[None, :] >= lens[:, None]
    tail[:5] = False
    H[tail] = 0
    H[0] = 0
    H[1, 0] = 0
    H[2, T - 1] = 0
    for k in range(c, T, c):
        H[3, [k - 1, k]] = 0
    cand = rng.integers(1, top, size=B)
    cand[4] = H[4, T // 2] = H[4, T - 1]
    cand[:4] = [top - 1, 1, top - 1, 2]
    neg = rng.integers(0, top, size=(B, max(T - 1, 0)))
    if past_2_24(case):
        special = np.array([ROUNDS_DOWN, EXACT, TWO24 - 1, ROUNDS_DOWN, 0])
        cand[5:10] = special
        for r in range(5, 10):
            pos = rng.choice(T, size=8, replace=False)
            H[r, pos] = np.resize(np.roll(special, r), 8)
            H[r, T - 1] = ROUNDS_DOWN
        H[6, 0] = EXACT
        neg[5:10, :4] = [ROUNDS_DOWN, EXACT, TWO24 - 1, 0]
    f["movieId"] = cand.astype(np.int32)
    for t, k in enumerate(history_keys(T)):
        f[k] = H[:, t].astype(np.int32)
    for j, k in enumerate(negative_history_keys(T)):
        f[k] = neg[:, j].astype(np.int32)
    f["label"] = (rng.random(B) < 0.4).astype(np.int32)
    return f


def f32_round(ids):
    """The float32 round trip every sequence kernel applies to a movie id."""
    return np.asarray(ids, np.int64).astype(np.float32).astype(np.int64)


MOVIE_KEYS = lambda T: ["movieId"] + history_keys(T) + negative_history_keys(T)


def touched_rows(case, f):
    """The sorted table rows `f`'s movie ids read, rounded through float32 or raw."""
    ids = np.concatenate([np.asarray(f[k]).astype(np.int64) for k in MOVIE_KEYS(case.T)])
    touched = np.unique(np.concatenate([f32_round(ids), ids]))
    assert touched[0] == 0
    return touched


def compact(case, f, W, raw=False):
    """(spec, weights, features) over a compact table of the rows `f` touches, in the rounded ids' order.  Ids
    are mapped through the float32 round trip (`raw`: not, the mutant of a kernel that reads raw ids) and
    `searchsorted`; 0 stays 0, the id DIEN masks.  Below 2^24 nothing changes."""
    if not past_2_24(case):
        return spec_of(case), W, f
    keys = MOVIE_KEYS(case.T)
    touched = touched_rows(case, f)
    Wc = dict(W, embedding=big_table_rows(touched, case.E))
    fc = dict(f)
    for k in keys:
        a = np.asarray(f[k]).astype(np.int64)
        fc[k] = np.searchsorted(touched, a if raw else f32_round(a)).astype(np.int32)
    return spec_of(case, vocab=len(touched)), Wc, fc


def logit_atol(case):
    return WIDE_LOGIT_ATOL if case.model == "dien" or case.E > 32 else LOGIT_ATOL


def oracle(case, W, f, defect=None, raw=False):
    """float64 (probabilities, logits) [B, 1] of the case, with an oracle mutant if `defect` is named."""
    spec, Wc, fc = compact(case, f, W, raw)
    if case.model == "din":
        return O.din_forward(spec, Wc, fc, np.float64, defect, chunk(case))
    return O.dien_forward(spec, Wc, fc, np.float64, defect)


def aux_oracle(case, W, f, defect=None):
    import test_dien_aux
    spec, Wc, fc = compact(case, f, W)
    return test_dien_aux.aux_oracle(spec, Wc, fc, defect)


def mutants(case):
    """The oracle mutants a case's kernel must be told apart from: name -> (kind, keyword arguments)."""
    out = {"position T - 1 dropped": dict(defect="last")}
    c = chunk(case)
    if case.model == "din":
        out["padding skipped in the pool"] = dict(defect="pad")
        if case.kernel == "din_kernel":
            if case.T % c:
                out["partial last chunk dropped"] = dict(defect="chunk")
            if case.T > c:
                out["alpha read at t mod %d" % c] = dict(defect="alpha")
    else:
        out["padding not masked"] = dict(defect="mask")
    if past_2_24(case):
        out["raw ids instead of their rounding"] = dict(raw=True)
    return out


FORWARD_CASES = [c for c in SEQ_MATRIX if c.kernel != "dien_train_step_kernel"]
FIT_CASES = [c for c in SEQ_MATRIX if c.kernel == "dien_train_step_kernel"]
_ids = lambda c: c.name


# ---- CPU: the table covers the dispatch, and reaches its edges ---------------------------------------------
def test_matrix_covers_every_instantiations_chunk_edges_and_ids_past_2_24():
    dispatched = dispatched_instantiations()
    assert {d[0] for d in dispatched} == {"din_kernel", "din_wg_kernel", "dien_kernel"}, dispatched
    assert {d for d in dispatched if d[0] == "dien_kernel"} >= {("dien_kernel", 12, True)}
    gaps = coverage_gaps(SEQ_MATRIX)
    assert not gaps, "SEQ_MATRIX lacks:\n" + "\n".join(gaps)


def test_the_guard_names_what_a_smaller_chunk_leaves_uncovered(tmp_path):
    """With kDinChunk = 16 in a copy of the sources, the guard names the T values 15, 16 and 17 at every EP."""
    for fname in ("din.cu", "din_wg.cu", "dien.cu", "kernels.h"):
        with open(os.path.join(CSRC, fname)) as f:
            src = f.read()
        if fname == "din.cu":
            src = src.replace("kDinChunk = %d;" % DIN_CHUNK, "kDinChunk = 16;")
        (tmp_path / fname).write_text(src)
    gaps = coverage_gaps(SEQ_MATRIX, str(tmp_path))
    assert gaps == ["din_kernel<%d>: no case at T = 15, 16, 17 (chunk 16)" % ep for ep in (12, 16, 32, 64)], gaps
    assert coverage_gaps([c for c in SEQ_MATRIX if c.kernel != "din_wg_kernel"]) == \
        ["din_wg_kernel: no case past 2^24"]


def test_matrix_cases_are_distinct():
    names = [c.name for c in SEQ_MATRIX]
    assert len(names) == len(set(names))


@pytest.mark.parametrize("case", SEQ_MATRIX, ids=_ids)
def test_case_inputs_reach_their_edges(case):
    T, c = case.T, chunk(case)
    f = features(case)
    H = history_of(case, f)
    cand = np.asarray(f["movieId"]).astype(np.int64)
    assert H.shape == (case.B, T) and case.B % 32 == 1            # one row past a 32-row tile
    assert np.all(H[0] == 0)                                       # all padding
    pad = H == 0
    assert any(pad[r, 0] and pad[r].sum() == 1 for r in range(case.B)) or T == 1
    assert any(pad[r, T - 1] and pad[r].sum() == 1 for r in range(case.B)) or T == 1
    for k in range(c, T, c):                                       # both sides of every chunk boundary
        assert any(pad[r, k - 1] and pad[r, k] and not pad[r].all() for r in range(case.B)), k
    assert any(cand[r] != 0 and cand[r] in H[r] for r in range(case.B))
    if case.kernel == "din_kernel" and T > c:                      # each position's own alpha
        alpha = weights(case)["au_prelu/alpha"]
        t = np.arange(c, T)
        assert np.all(np.any(alpha[t] != alpha[t % c], axis=1))
    W = weights(case)
    tab0 = big_table_rows([0], case.E)[0] if past_2_24(case) else W["embedding"][0]
    assert np.abs(tab0).min() >= 0.3                              # row 0 is clearly not a zero row
    if past_2_24(case):
        ids = np.concatenate([cand, H.ravel()])
        assert f32_round([ROUNDS_DOWN, EXACT, ROUNDS_OUT]).tolist() == [TWO24, EXACT, BIG_VOCAB]
        assert ROUNDS_DOWN in cand and ROUNDS_DOWN in H and EXACT in ids and TWO24 - 1 in ids and 0 in ids
        assert ROUNDS_OUT not in ids and np.all(f32_round(ids) < BIG_VOCAB)
        rows = big_table_rows([TWO24, ROUNDS_DOWN, ROUNDS_OUT], case.E)
        assert np.abs(rows[1] - rows[0]).max() > 0.1 and np.abs(rows[2] - rows[0]).max() > 0.1
        if case.model == "dien":
            neg = np.stack([np.asarray(f[k]) for k in negative_history_keys(T)], 1)
            assert ROUNDS_DOWN in neg


@functools.lru_cache(maxsize=None)
def mutant_shifts(case):
    """{mutant: the largest shift it gives a row, in units of the tolerance the GPU check holds that output to}:
    the logit for every mutant, aux for DIEN's aux sum without its last step."""
    W, f = weights(case), features(case)
    _, z = oracle(case, W, f)
    out = {}
    for name, kw in mutants(case).items():
        _, zd = oracle(case, W, f, **kw)
        out[name] = float(np.abs(zd - z).max() / logit_atol(case))
    if case.aux and case.T > 1:
        a, ad = aux_oracle(case, W, f), aux_oracle(case, W, f, defect="last")
        out["aux sum without its last step"] = float((np.abs(ad - a) / (AUX_ATOL + AUX_RTOL * np.abs(a))).max())
    return out


@pytest.mark.parametrize("case", FORWARD_CASES, ids=_ids)
def test_each_case_fails_every_mutant_that_applies(case):
    """Every oracle mutant of a defect the kernel could have moves some row past the case's tolerance."""
    weak = {k: v for k, v in mutant_shifts(case).items() if v <= 1.0}
    assert not weak, "mutants within the tolerance: %s" % weak


def test_each_kernel_has_a_case_ten_tolerances_from_every_mutant():
    """For each kernel (dien_kernel's AUX variant apart), each mutant moves some row of some case by more than 10x
    the tolerance.  Short DIEN histories sit closer (one padding row at T = 1; a 200-step GRU forgets its last
    step), so the 10x margin is asked of the kernel, not of every case."""
    best = collections.defaultdict(float)
    for case in FORWARD_CASES:
        for name, v in mutant_shifts(case).items():
            key = (case.kernel, case.aux, name)
            best[key] = max(best[key], v)
    want = {"din_kernel": {"position T - 1 dropped", "padding skipped in the pool", "partial last chunk dropped",
                           "alpha read at t mod %d" % DIN_CHUNK, "raw ids instead of their rounding"},
            "din_wg_kernel": {"raw ids instead of their rounding"},
            "dien_kernel": {"position T - 1 dropped", "padding not masked", "raw ids instead of their rounding"}}
    for kernel, aux in {(c.kernel, c.aux) for c in FORWARD_CASES}:
        names = want[kernel] | ({"aux sum without its last step"} if aux else set())
        for name in names:
            assert best[(kernel, aux, name)] > 10.0, (kernel, aux, name, best[(kernel, aux, name)])


def test_mutant_hooks_change_nothing_where_they_do_not_apply():
    """The "chunk" mutant at a whole number of chunks, and "alpha" within the first chunk, are the oracle."""
    for case in SEQ_MATRIX:
        if case.kernel == "din_kernel" and case.T in (32, 64) and not past_2_24(case) and case.E == 10:
            W, f = weights(case), features(case)
            _, z = oracle(case, W, f)
            assert np.array_equal(oracle(case, W, f, defect="chunk")[1], z)
        if case.kernel == "din_kernel" and case.T == 31 and case.E == 10:
            W, f = weights(case), features(case)
            assert np.array_equal(oracle(case, W, f, defect="alpha")[1], oracle(case, W, f)[1])
