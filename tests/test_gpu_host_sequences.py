"""Mixed call sequences on the host entry points of one model.

A serving process keeps one model and calls srs_predict_host, srs_rank_host and srs_rank_user_host on it in any
order, at request sizes that change from call to call.  All three use one private staging slot (`slots[kSlots]` in
csrc/model.cu), and each grows that slot's buffers by its own rule: the batch block (`ensure_slot`, first capacity
max(B, 1024)), the pinned completion record and result buffer (`ensure_done`, first capacity max(k, 1024)), the
rank scratch, and the request staging of srs_rank_user_host.  The ranking tail switches kernels at n = 1024
(`topk_small_kernel`) and at n = 4096 (`kSortChunk`).

Every call below is checked against a second model with the same weights that only runs srs_predict_device on a
fresh device batch of the same rows: the scores must be the same bits, a ranking must equal `O.rank_topk` of those
scores, and a sample of at most 256 rows must match the float64 oracle.

* GPU:
  - `SCRIPT`: every ordered pair of the five synchronous-slot calls on a fresh model, the second call growing the slot;
  - a seeded random walk of 150 calls per model, with one out-of-range id in one row at fixed steps;
  - the error words of the host slots and of the device path do not leak into each other;
  - srs_rank_host and srs_predict_host_batches reject a bad argument before their first launch;
  - srs_rank_user_host through the raw ABI: history lengths, genres below -1, duplicate candidates, a table upload
    that fails;
  - two threads on one model give the bits of a serial run.
* CPU: `SCRIPT` runs each entry point at and one past every size threshold read from the sources, and covers every
  ordered pair; the Python statement of the request assembly agrees with `featurestore.assemble`.
"""
import ctypes as C
import itertools
import os
import re
import threading
import zlib

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import ctr_oracle as O
from sparrowrecsys_b200 import _lib
from sparrowrecsys_b200 import featurestore as FS
from sparrowrecsys_b200.features import encode_batch, genre_to_index, synthetic_features
from sparrowrecsys_b200.spec import MOVIE_GENRE_KEYS, USER_GENRE_KEYS, default_spec, history_keys
from sparrowrecsys_b200.weights import init_weights
from test_gpu_kernel_matrix import CSRC, LOGIT_ATOL, PROB_ATOL

# ---- the script ---------------------------------------------------------------------------------------------
# the calls that use the private slot: srs_predict_host in its three modes, srs_rank_host, srs_rank_user_host
ENTRY_FUNCS = {"srs_predict_host": ("host", "host_pinned", "host_pinned_mixed"),
               "srs_rank_host": ("rank",), "srs_rank_user_host": ("rank_user",)}
ENTRY_POINTS = ("host",               # pageable probs and logits: the general path
                "host_pinned",        # pinned probs and logits: the latency path (kernel writes the host buffers)
                "host_pinned_mixed",  # pinned probs, pageable logits: falls back to the general path
                "rank", "rank_user")
RANKING = ("rank", "rank_user")
# (n_a, k_a, n_b, k_b): the second call's n exceeds the capacity the first call leaves
PATTERNS = [(1024, 1024, 1025, 1025),
            (0, 0, 4096, 1024),
            (1025, 0, 4097, 4102),
            (4096, 4101, 4097, 1),
            (800, 800, 6000, 0)]
SCRIPT = [(a, na, ka, b, nb, kb)
          for i, a in enumerate(ENTRY_POINTS) for j, b in enumerate(ENTRY_POINTS)
          for na, ka, nb, kb in [PATTERNS[(i + j) % len(PATTERNS)]]]

WALK_STEPS = 150
WALK_ENTRY_POINTS = ENTRY_POINTS + ("batches", "async")
BAD_EVERY = 10                     # one out-of-range id at steps 9, 19, ...
MAX_N = 10000

# name -> (model, spec overrides, narrow_ids, kernel)
MODELS = {
    "din": ("din", dict(emb_dim=32, hist_len=50, n_movies=20000, n_users=3000), False, "din_wg_kernel"),
    "din_narrow": ("din", dict(emb_dim=32, hist_len=50, n_movies=20000, n_users=3000), True, "din_wg_kernel"),
    "widendeep": ("widendeep", dict(emb_dim=10, n_movies=3000, n_users=3000), False, "embmlp_tc_kernel<wide&deep>"),
    "neuralcf": ("neuralcf", dict(n_movies=3000, n_users=3000), False, "ncf_kernel<neural_cf_model_1>"),
}
CSV = os.path.join(GOLDEN, "samples_head.csv")


def _hist_cols(spec):
    return spec.hist_len if spec.model in ("din", "dien") else (1 if spec.model == "widendeep" else 0)


def _dense(spec):
    return spec.model not in ("neuralcf", "twotowers")


def request_features(spec, user, cand, genres, nums):
    """Statement of srs_rank_user_host's request assembly (assemble_request_kernel) as a feature dict: the user
    columns broadcast to every row, the movie columns gathered from the table arrays (genres [rows, 3], numerics
    [rows, 4]), the history padded with id 0, genres below 0 read as -1 (missing)."""
    cand = np.asarray(cand, np.int32).reshape(-1)
    n = cand.shape[0]
    f = {"movieId": cand, "userId": np.full(n, user["user_id"], np.int32)}
    keys = history_keys(spec.hist_len) if spec.model in ("din", "dien") else ["userRatedMovie1"]
    hist = list(user["hist"])
    for t, key in enumerate(keys[:_hist_cols(spec)]):
        f[key] = np.full(n, hist[t] if t < len(hist) else 0, np.int32)
    for j, key in enumerate(USER_GENRE_KEYS):
        f[key] = np.full(n, max(int(user["genres"][j]), -1), np.int32)
    for j, key in enumerate(("userAvgRating", "userRatingCount", "userRatingStddev")):
        f[key] = np.full(n, user["nums"][j], np.float32)
    if _dense(spec):
        g = np.maximum(genres[cand], -1)
        for j, key in enumerate(MOVIE_GENRE_KEYS):
            f[key] = g[:, j].astype(np.int32)
        for j, key in enumerate(("movieAvgRating", "movieRatingCount", "movieRatingStddev", "releaseYear")):
            f[key] = nums[cand, j].astype(np.float32)
    return f


def table_arrays(table):
    """A MovieFeatureTable as the arrays CTRModel.set_movie_table uploads."""
    genres = np.stack([table.idx_cols[k] for k in MOVIE_GENRE_KEYS], axis=1).astype(np.int32)
    nums = np.stack([table.float_cols["movieAvgRating"], table.int_cols["movieRatingCount"].astype(np.float32),
                     table.float_cols["movieRatingStddev"], table.int_cols["releaseYear"].astype(np.float32)],
                    axis=1).astype(np.float32)
    return genres, nums


def user_row(spec, fields):
    """A `uf:` hash as the srs_user_row CTRModel.rank_user sends."""
    hc = _hist_cols(spec)
    typed = FS.parse_user_features(fields, max(hc, 1))
    keys = history_keys(spec.hist_len) if spec.model in ("din", "dien") else ["userRatedMovie1"]
    genres = [int(genre_to_index([typed["userGenre%d" % (g + 1)]])[0]) for g in range(5)]
    nums = np.array([typed["userAvgRating"], np.float32(typed["userRatingCount"]), typed["userRatingStddev"]],
                    np.float32)
    return dict(user_id=0, genres=genres, nums=nums, hist=np.array([typed[k] for k in keys[:hc]], np.int32))


# ---- CPU: the script reaches every threshold and every ordered pair -----------------------------------------
def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _function(src, name):
    """Source of the C function `name`, from its signature to its closing brace in column 0."""
    found = re.findall(r"^(?:int|cudaError_t) %s\(.*?^\}" % name, src, re.M | re.S)
    assert len(found) == 1, name
    return found[0]


def size_thresholds():
    """{"n": {what: threshold}, "k": {what: threshold}}, read from csrc/model.cu and csrc/topk.cu."""
    model, topk = _source("model.cu"), _source("topk.cu")
    found = {
        ("n", "ensure_slot first capacity"): re.findall(r"std::max\(B, (\d+)\)", _function(model, "ensure_slot")),
        ("n", "topk_small_kernel limit"): re.findall(r"if \(n <= (\d+)\)", _function(topk, "launch_topk_done")),
        ("n", "kSortChunk"): re.findall(r"constexpr int kSortChunk = (\d+);", topk),
        ("k", "ensure_done first capacity"): re.findall(r"std::max\(k, (\d+)\)", _function(model, "ensure_done")),
    }
    out = {"n": {}, "k": {}}
    for (axis, what), values in found.items():
        assert len(values) == 1, "%s: expected one match, found %s" % (what, values)
        out[axis][what] = int(values[0])
    return out


def slot_entry_points():
    """The exported functions of csrc/model.cu that use the private slot."""
    return {name for name, body in re.findall(r"^int (srs_\w+)\((.*?)^\}", _source("model.cu"), re.M | re.S)
            if "slots[kSlots]" in body}


def script_calls():
    return [c for a, na, ka, b, nb, kb in SCRIPT for c in ((a, na, ka), (b, nb, kb))]


def test_script_runs_every_entry_point_at_and_past_every_threshold():
    assert slot_entry_points() == set(ENTRY_FUNCS), "a new entry point on the private slot needs script cases"
    assert set(ENTRY_POINTS) == {ep for eps in ENTRY_FUNCS.values() for ep in eps}
    th = size_thresholds()
    calls = script_calls()
    for ep in ENTRY_POINTS:
        ns = {n for e, n, _ in calls if e == ep}
        assert 0 in ns, "%s never runs an empty batch" % ep
        for what, t in th["n"].items():
            assert {t, t + 1} <= ns, "%s never runs n = %d and n = %d (%s)" % (ep, t, t + 1, what)
        if ep in RANKING:
            ks = {min(k, n) for e, n, k in calls if e == ep}
            for what, t in th["k"].items():
                assert {t, t + 1} <= ks, "%s never runs k = %d and k = %d (%s)" % (ep, t, t + 1, what)
            assert any(k == 0 < n for e, n, k in calls if e == ep), "%s never runs k = 0" % ep
            assert any(k > n > 0 for e, n, k in calls if e == ep), "%s never runs k > n" % ep


def test_script_covers_every_ordered_pair_and_grows_the_slot():
    cap0 = size_thresholds()["n"]["ensure_slot first capacity"]
    assert sorted((a, b) for a, _, _, b, _, _ in SCRIPT) == sorted(itertools.product(ENTRY_POINTS, repeat=2))
    for a, na, _, b, nb, _ in SCRIPT:
        cap = max(na, cap0) if na > 0 else 0
        assert nb > cap, (a, na, b, nb)


@pytest.mark.parametrize("model,kw", [("din", dict(emb_dim=32, hist_len=50)), ("widendeep", {}), ("neuralcf", {})])
def test_request_statement_matches_featurestore_assemble(model, kw):
    """The feature dict the GPU tests expect srs_rank_user_host to assemble equals, after encoding, the one
    `featurestore.assemble(..., encoded=True)` builds from the same `uf:` / `mf:` hashes."""
    store = FS.FeatureStore.from_samples(CSV)
    raw = FS.read_sample_strings(CSV)
    spec = default_spec(model, **kw)
    table = FS.MovieFeatureTable.from_store(store, spec.n_movies)
    genres, nums = table_arrays(table)
    T = spec.hist_len if model == "din" else 5
    cand = store.movie_ids()[:50] + [spec.n_movies - 1, 0, 7]          # the last three: no hash, defaults
    all_users = list(dict.fromkeys(raw["userId"]))
    short = [u for u in all_users if store.user_features(int(u)).get("userRatedMovie5", "") == ""][:2]
    assert short, "the samples should include users with short histories"
    for uid in [int(u) for u in all_users[:6] + short]:
        fields = store.user_features(uid)
        user = dict(user_row(spec, fields), user_id=uid)
        a = encode_batch(spec, request_features(spec, user, cand, genres, nums))
        b = encode_batch(spec, FS.assemble(uid, fields, cand, table, hist_len=T, encoded=True))
        for name in ("movie_id", "user_id", "hist", "movie_genre", "user_genre", "numerics"):
            x, y = getattr(a, name), getattr(b, name)
            assert (x is None and y is None) or np.array_equal(x, y), (model, uid, name)


# ---- GPU ------------------------------------------------------------------------------------------------------
def _last_error():
    return _lib.load().srs_last_error().decode("utf-8", "replace")


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _pinned(n):
    import torch
    return torch.full((max(n, 1),), float("nan"), dtype=torch.float32, pin_memory=True)


def _launches(fn):
    from sparrowrecsys_b200.model import launch_count
    before = launch_count()
    r = fn()
    return r, launch_count() - before


class Rig:
    """One model kind: spec, weights, movie table, and the reference model, which only runs srs_predict_device."""

    def __init__(self, name):
        from sparrowrecsys_b200.model import CTRModel
        model, over, self.narrow, self.kernel = MODELS[name]
        self.name = name
        self.spec = spec = default_spec(model, **over)
        self.seed = zlib.crc32(name.encode()) & 0xFFFF
        self.W = init_weights(spec, zlib.crc32(model.encode()) & 0xFFFF)
        self.hc = _hist_cols(spec)
        self.dense = _dense(spec)
        rows = int(spec.n_movies * 0.8)                 # fewer rows than the vocabulary
        rng = np.random.default_rng(self.seed)
        self.genres = rng.integers(0, spec.n_genres, (rows, 3)).astype(np.int32)
        self.genres[rng.random((rows, 3)) < 0.2] = -1
        self.nums = np.stack([rng.uniform(0.5, 5.0, rows).round(2), rng.integers(1, 30000, rows),
                              rng.uniform(0.0, 2.0, rows).round(2), rng.integers(1900, 2016, rows)],
                             axis=1).astype(np.float32)
        self.table_rows = rows
        self.cand_limit = rows if self.dense else spec.n_movies
        self.ref = CTRModel(spec, self.W)
        self.lib = _lib.load()

    def model(self):
        from sparrowrecsys_b200.model import CTRModel
        m = CTRModel(self.spec, self.W, narrow_ids=self.narrow)
        assert m.kernel_name == self.kernel
        assert self.narrow == m.narrow_ids
        _lib.check(self.lib.srs_model_set_movie_features(m._h, self.table_rows, self.genres.ctypes.data,
                                                         self.nums.ctypes.data))
        return m

    def bad_kinds(self):
        kinds = ["movie", "user"]
        if self.hc:
            kinds.append("hist")
        if self.dense:
            kinds += ["genre", "cand_table_end"]
        return kinds + ["cand_vocab_end"]

    def user(self, rng, n_hist=None):
        n_hist = self.hc if n_hist is None else n_hist
        return dict(user_id=int(rng.integers(0, self.spec.n_users)),
                    genres=[int(g) for g in rng.integers(-1, self.spec.n_genres, 5)],
                    nums=np.array([rng.uniform(0.5, 5.0), rng.integers(0, 3000), rng.uniform(0.0, 2.0)], np.float32),
                    hist=rng.integers(0, self.spec.n_movies, n_hist).astype(np.int32))

    def features(self, n, seed):
        f = synthetic_features(self.spec, max(n, 2), seed=seed)
        f["movieId"][-1], f["userId"][-1] = self.spec.n_movies - 1, self.spec.n_users - 1
        return {k: np.asarray(v)[:n] for k, v in f.items()}

    def ref_scores(self, enc):
        """(probs, logits) of srs_predict_device on a fresh device batch of `enc`'s rows."""
        import torch
        if enc.B == 0:
            return np.empty(0, np.float32), np.empty(0, np.float32)
        d = self.ref.to_device(enc)
        p = torch.full((enc.B,), float("nan"), dtype=torch.float32, device="cuda:0")
        z = torch.full_like(p, float("nan"))
        self.ref.predict_device(d, p, z)
        self.ref.status()
        return p.cpu().numpy(), z.cpu().numpy()


class Call:
    """One call of an entry point with its inputs, run on a model and checked against the reference.
    `bad`: one out-of-range id of that kind goes into row n // 2 of what the call sends."""

    def __init__(self, rig, ep, n, k, seed, bad=None, logits=True, probs=True, n_hist=None, user=None, cand=None):
        self.ep, self.n, self.k, self.bad, self.seed = ep, n, k, bad, seed
        self.want_logits = logits or ep == "host_pinned_mixed"     # pageable logits are what make that mode
        self.want_probs = probs
        spec = rig.spec
        rng = np.random.default_rng(seed)
        self.bad_row = n // 2 if bad and n > 0 else None
        self.chunks = [(0, n)]
        if ep == "rank_user":
            self.user = user if user is not None else rig.user(rng, n_hist)
            self.cand = (np.asarray(cand, np.int32) if cand is not None
                         else rng.integers(0, rig.cand_limit, n).astype(np.int32))
            ref_cand = self.cand.copy()
            if self.bad_row is not None:
                assert bad in ("cand_table_end", "cand_vocab_end")
                self.cand[self.bad_row] = rig.table_rows if bad == "cand_table_end" else spec.n_movies
                ref_cand[self.bad_row] = 0
            self.feats = request_features(spec, self.user, ref_cand, rig.genres, rig.nums)
            self.enc_ref = encode_batch(spec, self.feats)
            return
        self.feats = rig.features(n, seed)
        self.enc_ref = encode_batch(spec, self.feats)
        self.enc = encode_batch(spec, self.feats, narrow_ids=rig.narrow)
        if self.bad_row is not None:
            r = self.bad_row
            if bad == "movie":
                self.enc.movie_id[r] = spec.n_movies
            elif bad == "user":
                self.enc.user_id[r] = -1
            elif bad == "hist":
                self.enc.hist[r, -1] = spec.n_movies
            elif bad == "genre":
                self.enc.user_genre[r, 0] = spec.n_genres
            else:
                raise AssertionError(bad)
        if ep in ("batches", "async") and n > 0:
            parts = int(rng.integers(1, 7 if ep == "batches" else 3))
            cuts = np.sort(rng.integers(0, n + 1, parts - 1)).tolist()
            self.chunks = list(zip([0] + cuts, cuts + [n]))
            self.slots = [int(s) for s in rng.permutation(4)[:len(self.chunks)]]

    def __repr__(self):
        return "%s(n=%d, k=%d, bad=%s, seed=%d)" % (self.ep, self.n, self.k, self.bad, self.seed)

    def _row(self):
        row = _lib.SrsUserRow()
        row.user_id = self.user["user_id"]
        for g in range(5):
            row.user_genre[g] = int(self.user["genres"][g])
        for j in range(3):
            row.user_numerics[j] = float(self.user["nums"][j])
        hist = np.ascontiguousarray(self.user["hist"], np.int32)
        row.n_hist = hist.shape[0]
        row.hist = hist.ctypes.data if hist.shape[0] else None
        return row, hist

    def run(self, lib, m):
        """Make the call; returns {"rc": [...], "probs", "logits" | "idx", "top", "probs", "launches"}."""
        from sparrowrecsys_b200.model import _host_struct
        n, k, h = self.n, self.k, m._h
        keep = []
        if self.ep in RANKING:
            idx = np.full(max(k, 1), -7, np.int32)
            top = np.full(max(k, 1), np.nan, np.float32)
            probs = np.full(max(n, 1), np.nan, np.float32) if self.want_probs else None
            if self.ep == "rank":
                b = _host_struct(self.enc, keep)
                rc, launches = _launches(lambda: lib.srs_rank_host(h, C.byref(b), k, idx.ctypes.data,
                                                                   top.ctypes.data))
                probs = None
            else:
                row, hist = self._row()
                rc, launches = _launches(lambda: lib.srs_rank_user_host(
                    h, C.byref(row), self.cand.ctypes.data if n else None, n, k, idx.ctypes.data,
                    top.ctypes.data, None if probs is None else probs.ctypes.data))
            kk = min(k, n)
            return dict(rc=[rc], idx=idx[:kk].copy(), top=top[:kk].copy(),
                        probs=None if probs is None else probs[:n].copy(), launches=launches)
        pinned_p = self.ep in ("host_pinned", "host_pinned_mixed", "async")
        pinned_z = self.ep == "host_pinned"
        tp = _pinned(n) if pinned_p else None
        tz = _pinned(n) if pinned_z and self.want_logits else None
        P = tp.numpy() if pinned_p else np.full(max(n, 1), np.nan, np.float32)
        Z = None
        if self.want_logits:
            Z = tz.numpy() if pinned_z else np.full(max(n, 1), np.nan, np.float32)
        zp = lambda lo: None if Z is None else Z.ctypes.data + 4 * lo
        if self.ep in ENTRY_POINTS:
            b = _host_struct(self.enc, keep)
            rc, launches = _launches(lambda: [lib.srs_predict_host(h, C.byref(b), P.ctypes.data, zp(0))])
        elif self.ep == "batches":
            nb = len(self.chunks)
            structs = (_lib.SrsBatch * nb)(*[_host_struct(self.enc.slice(lo, hi), keep) for lo, hi in self.chunks])
            pp = (C.c_void_p * nb)(*[P.ctypes.data + 4 * lo for lo, _ in self.chunks])
            lp = None if Z is None else (C.c_void_p * nb)(*[zp(lo) for lo, _ in self.chunks])
            rc, launches = _launches(lambda: [lib.srs_predict_host_batches(h, nb, structs, pp, lp)])
        else:
            structs = [_host_struct(self.enc.slice(lo, hi), keep) for lo, hi in self.chunks]

            def go():
                rcs = [lib.srs_predict_host_async(h, s, C.byref(b), P.ctypes.data + 4 * lo, zp(lo))
                       for (lo, _), s, b in zip(self.chunks, self.slots, structs)]
                return rcs + [lib.srs_wait_slot(h, s) for s in reversed(self.slots)]
            rc, launches = _launches(go)
        return dict(rc=rc, probs=P[:n].copy(), logits=None if Z is None else Z[:n].copy(), launches=launches)

    def expected_rc(self):
        bad = self.bad_row is not None
        if self.ep != "async" or self.n == 0:
            return [_lib.SRS_ERR_RANGE if bad else _lib.SRS_OK]
        waits = [_lib.SRS_ERR_RANGE if bad and lo <= self.bad_row < hi else _lib.SRS_OK
                 for lo, hi in reversed(self.chunks)]
        return [_lib.SRS_OK] * len(self.chunks) + waits

    def check(self, rig, out):
        what = "%s on %s" % (self, rig.name)
        assert out["rc"] == self.expected_rc(), "%s: rc %s (%s)" % (what, out["rc"], _last_error())
        n = self.n
        if n == 0:
            return
        ref_p, ref_z = np.empty(n, np.float32), np.empty(n, np.float32)
        ref_launches = 0
        for lo, hi in self.chunks:
            (p, z), d = _launches(lambda: rig.ref_scores(self.enc_ref.slice(lo, hi)))
            ref_p[lo:hi], ref_z[lo:hi] = p, z
            ref_launches += d
        good = np.ones(n, bool)
        if self.bad_row is not None:
            good[self.bad_row] = False
        if out.get("probs") is not None:
            assert _same_bits(out["probs"][good], ref_p[good]), "%s: scores differ from the reference" % what
        if out.get("logits") is not None:
            assert _same_bits(out["logits"][good], ref_z[good]), "%s: logits differ from the reference" % what
        if self.ep in ENTRY_POINTS and self.ep not in RANKING:
            # the latency path adds the completion kernel; narrow ids add the widening kernel
            extra = (1 if rig.narrow else 0) + (1 if self.ep == "host_pinned" else 0)
            assert out["launches"] == ref_launches + extra, "%s: %d launches, expected %d" % (
                what, out["launches"], ref_launches + extra)
        if self.ep in RANKING and self.bad_row is None:
            ridx, rtop = O.rank_topk(ref_p, self.k)
            assert np.array_equal(out["idx"], ridx), "%s: ranking differs from the reference" % what
            assert _same_bits(out["top"], rtop), "%s: ranked scores differ from the reference" % what
        rows = np.flatnonzero(good)
        if rows.size == 0:
            return
        if rows.size > 256:
            rows = np.sort(np.random.default_rng(self.seed).choice(rows, 256, replace=False))
        po, zo = O.forward(rig.spec, rig.W, {k: np.asarray(v)[rows] for k, v in self.feats.items()},
                           dtype=np.float64)
        assert np.abs(ref_p[rows] - po[:, 0]).max() <= PROB_ATOL, what
        assert np.abs(ref_z[rows] - zo[:, 0]).max() <= LOGIT_ATOL, what

    def __call__(self, rig, m):
        out = self.run(rig.lib, m)
        self.check(rig, out)
        return out


def _assert_status_clean(rig, m, what):
    rc = rig.lib.srs_model_status(m._h)
    assert rc == _lib.SRS_OK, "%s: status %d (%s)" % (what, rc, _last_error())


def _pair_id(p):
    return "%s%d-%s%d" % (p[0], p[1], p[3], p[4])


@pytest.fixture(scope="module", params=list(MODELS))
def rig(request):
    r = Rig(request.param)
    yield r
    r.ref.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pair", SCRIPT, ids=_pair_id)
def test_second_call_grows_the_slot_after_the_first(rig, pair):
    a, na, ka, b, nb, kb = pair
    with rig.model() as m:
        Call(rig, a, na, ka, seed=rig.seed + 1)(rig, m)
        Call(rig, b, nb, kb, seed=rig.seed + 2)(rig, m)
        Call(rig, a, 300, 17, seed=rig.seed + 3)(rig, m)          # and the first entry point again, on the grown slot
        _assert_status_clean(rig, m, "after %s" % _pair_id(pair))


def walk_plan(rig):
    """(entry point, n, k, bad kind or None, want logits / probs, seed) for each step of the random walk."""
    rng = np.random.default_rng(rig.seed + 99)
    kinds = rig.bad_kinds()
    host_eps = [ep for ep in WALK_ENTRY_POINTS if ep != "rank_user"]
    plan, n_host_bad = [], 0
    for step in range(WALK_STEPS):
        n = int(np.clip(np.round(np.exp(rng.uniform(0.0, np.log(MAX_N)))), 1, MAX_N))
        k = [0, 1, int(rng.integers(0, n + 1)), n, n + 5][int(rng.integers(5))]
        bad = None
        if step % BAD_EVERY == BAD_EVERY - 1:
            j = step // BAD_EVERY
            bad = kinds[j % len(kinds)]
            if bad.startswith("cand"):
                ep = "rank_user"
            else:
                ep, n_host_bad = host_eps[n_host_bad % len(host_eps)], n_host_bad + 1
        else:
            ep = WALK_ENTRY_POINTS[int(rng.integers(len(WALK_ENTRY_POINTS)))]
        plan.append((ep, n, k, bad, bool(rng.integers(2)), int(rng.integers(1 << 30))))
    return plan


@pytest.mark.gpu
def test_random_walk_matches_the_reference(rig):
    plan = walk_plan(rig)
    assert {b for _, _, _, b, _, _ in plan if b} == set(rig.bad_kinds())
    assert {ep for ep, _, _, b, _, _ in plan if b} == set(WALK_ENTRY_POINTS)
    with rig.model() as m:
        for step, (ep, n, k, bad, extra, seed) in enumerate(plan):
            Call(rig, ep, n, k, seed, bad=bad, logits=extra, probs=extra or ep == "rank")(rig, m)
            if bad:
                # the error word was consumed by the bad call: the next call of every entry point is clean
                for i, ep2 in enumerate(WALK_ENTRY_POINTS):
                    Call(rig, ep2, 37 + i, 5, seed + 1 + i)(rig, m)
                _assert_status_clean(rig, m, "after the bad step %d (%s, %s)" % (step, ep, bad))
        _assert_status_clean(rig, m, "after the walk")


@pytest.mark.gpu
def test_error_words_stay_with_their_path(rig):
    """A bad device batch latches only the device word, which srs_model_status reports; a bad host call raises
    itself and leaves nothing for the device path or srs_model_status."""
    import torch
    spec = rig.spec
    with rig.model() as m:
        enc = encode_batch(spec, rig.features(700, rig.seed + 5))
        enc.movie_id[3] = spec.n_movies
        out = torch.empty(700, dtype=torch.float32, device="cuda:0")
        m.predict_device(m.to_device(enc), out)
        torch.cuda.synchronize()
        for i, ep in enumerate(WALK_ENTRY_POINTS):
            Call(rig, ep, 1500 + 100 * i, 20, rig.seed + 10 + i)(rig, m)
        with pytest.raises(ValueError):
            m.status()
        m.status()                                                     # cleared by the report
        for i, ep in enumerate(WALK_ENTRY_POINTS):
            bad = "cand_vocab_end" if ep == "rank_user" else "user"
            Call(rig, ep, 900, 3, rig.seed + 20 + i, bad=bad)(rig, m)
            _assert_status_clean(rig, m, "after a bad %s call" % ep)
            good = encode_batch(spec, rig.features(64, rig.seed + 30 + i))
            out = torch.empty(64, dtype=torch.float32, device="cuda:0")
            m.predict_device(m.to_device(good), out)
            _assert_status_clean(rig, m, "device batch after a bad %s call" % ep)
            assert _same_bits(out.cpu().numpy(), rig.ref_scores(good)[0])


@pytest.mark.gpu
def test_rank_host_rejects_a_null_top_idx_before_it_launches(rig):
    """srs_rank_host with k > 0 and no top_idx fails before it stages the batch, so an out-of-range id in that
    batch leaves no error word behind for the next call on the private slot."""
    from sparrowrecsys_b200.model import _host_struct
    with rig.model() as m:
        keep = []
        b = _host_struct(Call(rig, "rank", 600, 5, rig.seed + 80, bad="user").enc, keep)
        top = np.full(5, np.nan, np.float32)
        rc, launches = _launches(lambda: rig.lib.srs_rank_host(m._h, C.byref(b), 5, None, top.ctypes.data))
        assert rc == _lib.SRS_ERR_INVALID, _last_error()
        assert launches == 0
        for i, ep in enumerate(("host", "host_pinned", "rank", "rank_user")):
            Call(rig, ep, 300, 5, rig.seed + 81 + i)(rig, m)
        _assert_status_clean(rig, m, "after the rejected srs_rank_host")


@pytest.mark.gpu
def test_predict_host_batches_checks_every_batch_before_it_launches(rig):
    """A srs_predict_host_batches call whose batch 1 has no movie_id fails before batch 0, which holds an
    out-of-range id, is launched: the next call and srs_model_status are clean."""
    from sparrowrecsys_b200.model import _host_struct
    with rig.model() as m:
        keep = []
        calls = [Call(rig, "host", 500, 0, rig.seed + 90, bad="user"), Call(rig, "host", 400, 0, rig.seed + 91)]
        structs = (_lib.SrsBatch * 2)(*[_host_struct(c.enc, keep) for c in calls])
        structs[1].movie_id = None
        out = [np.full(c.n, np.nan, np.float32) for c in calls]
        pp = (C.c_void_p * 2)(*[p.ctypes.data for p in out])
        rc, launches = _launches(lambda: rig.lib.srs_predict_host_batches(m._h, 2, structs, pp, None))
        assert rc == _lib.SRS_ERR_INVALID, _last_error()
        assert launches == 0
        Call(rig, "batches", 700, 0, rig.seed + 92)(rig, m)
        _assert_status_clean(rig, m, "after the rejected srs_predict_host_batches")


@pytest.mark.gpu
def test_rank_user_request_edges(rig):
    spec, T = rig.spec, rig.hc
    rng = np.random.default_rng(rig.seed + 40)
    with rig.model() as m:
        for i, n_hist in enumerate(sorted({0, min(1, T), max(T - 1, 0), T})):
            Call(rig, "rank_user", 900, 10, rig.seed + 41 + i, n_hist=n_hist)(rig, m)
        # genres below -1 are read as -1 (missing)
        user = dict(rig.user(rng), genres=[-3, -1, 4, -2, spec.n_genres - 1])
        Call(rig, "rank_user", 500, 20, rig.seed + 50, user=user)(rig, m)
        # duplicate candidates: equal scores rank by position, in every branch of the ranking tail
        for i, n in enumerate((700, 3000, 5000)):
            cand = rng.choice(rng.integers(0, rig.cand_limit, 12), n).astype(np.int32)
            Call(rig, "rank_user", n, n, rig.seed + 51 + i, cand=cand)(rig, m)
        # a table upload that fails on its last row leaves the previous table in place
        call = Call(rig, "rank_user", 2000, 50, rig.seed + 60)
        before = call(rig, m)
        genres = (rig.genres + 1) % spec.n_genres
        genres[-1, 2] = spec.n_genres
        nums = rig.nums + np.float32(1)
        rc = rig.lib.srs_model_set_movie_features(m._h, rig.table_rows, genres.ctypes.data, nums.ctypes.data)
        assert rc == _lib.SRS_ERR_RANGE, _last_error()
        after = call(rig, m)
        for key in ("idx", "top", "probs"):
            assert _same_bits(before[key], after[key]), key
        _assert_status_clean(rig, m, "after the failed upload")


@pytest.mark.gpu
def test_two_threads_on_one_model_match_a_serial_run(rig):
    """predict_host, rank_host, rank_user and predict_host_batches hold the model's lock: two threads calling
    them on one model (ctypes releases the GIL) get the bits of the same calls made one after another."""
    eps = ("host", "host_pinned", "rank", "rank_user", "batches")
    plans = []
    for t in range(2):
        rng = np.random.default_rng(rig.seed + 70 + t)
        plan = []
        for i in range(15):
            n = int(np.clip(np.round(np.exp(rng.uniform(0.0, np.log(8000)))), 1, 8000))
            plan.append(Call(rig, eps[(i + t) % len(eps)], n, int(rng.integers(0, n + 6)), int(rng.integers(1 << 30))))
        plans.append(plan)
    with rig.model() as m:
        serial = [[c(rig, m) for c in plan] for plan in plans]
        results, errors = [None, None], []
        barrier = threading.Barrier(2)

        def work(t):
            try:
                barrier.wait()
                results[t] = [c.run(rig.lib, m) for c in plans[t]]
            except BaseException as e:          # reported below, on the main thread
                errors.append(e)
        threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert not errors, errors
        for t in range(2):
            for c, a, b in zip(plans[t], serial[t], results[t]):
                assert a["rc"] == b["rc"], (t, c)
                for key in ("probs", "logits", "idx", "top"):
                    if a.get(key) is not None:
                        assert _same_bits(a[key], b[key]), (t, c, key)
        _assert_status_clean(rig, m, "after the threads")
