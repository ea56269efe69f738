"""Host-side mirror of the reference's model-call surface over the C ABI.

The reference's callable is a module-level Keras `model` and the call is
`model.predict(feature_dict) -> float32[N,1]` (e.g.
`TFRecModel/src/com/sparrowrecsys/offline/tensorflow/DIN.py:169,185`); at serve
time the same graph answers TF-Serving's `:predict`
(`online/recprocess/RecForYouProcess.java:113-138`).  `CTRModel` keeps that
surface - same key names, same dtypes, unknown keys ignored, `KeyError` for a
missing key, `ValueError` for an out-of-range id (TF's identity-column assert) -
and forwards to `libsrs_ctr.so` through ctypes.  There is no fallback: without the
CUDA library or a GPU, construction raises.

PyTorch appears only in the `*_device` helpers, as the on-device container.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Optional

import numpy as np

from . import _lib
from .features import EncodedBatch, _as_ids, encode_batch, negative_history_keys
from .spec import ModelSpec, default_spec
from .weights import aux_weight_shapes, check_weights, has_aux_weights, init_weights, weight_shapes


def _spec_struct(spec: ModelSpec) -> _lib.SrsSpec:
    s = _lib.SrsSpec()
    s.kind = spec.kind
    s.emb_dim = spec.emb_dim
    s.n_movies = spec.n_movies
    s.n_users = spec.n_users
    s.n_genres = spec.n_genres
    s.hist_len = spec.hist_len
    s.n_hidden = len(spec.hidden)
    for i, h in enumerate(spec.hidden):
        s.hidden[i] = h
    s.au_hidden = spec.au_hidden
    s.cross_buckets = spec.cross_buckets
    s.proj_dim = spec.proj_dim
    s.final_dense = 1 if spec.final_dense else 0
    return s


class DeviceBatch:
    """An encoded batch resident in HBM (torch tensors as containers)."""

    def __init__(self, enc: EncodedBatch, device, hist_cols: int):
        import torch
        dev = torch.device(device)
        t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        self.B = enc.B
        self.movie_id = t(enc.movie_id)
        self.user_id = t(enc.user_id)
        self.hist = t(None if enc.hist is None else enc.hist.astype(np.int32, copy=False))
        self.movie_genre = t(enc.movie_genre)
        self.user_genre = t(enc.user_genre)
        self.numerics = t(enc.numerics)
        self.hist_stride = 0 if enc.hist is None else enc.hist.shape[1]

    def struct(self) -> _lib.SrsBatch:
        p = lambda x: None if x is None else x.data_ptr()
        return _lib.SrsBatch(self.B, self.hist_stride, p(self.movie_id), p(self.user_id),
                             p(self.hist), p(self.movie_genre), p(self.user_genre),
                             p(self.numerics))


def _host_struct(enc: EncodedBatch, keep: list) -> _lib.SrsBatch:
    def p(a, dtype):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=dtype)
        keep.append(a)
        return a.ctypes.data
    hs = 0 if enc.hist is None else enc.hist.shape[1]
    narrow = enc.hist is not None and enc.hist.dtype == np.uint16      # srs_batch::hist16
    return _lib.SrsBatch(enc.B, hs, p(enc.movie_id, np.int32), p(enc.user_id, np.int32),
                         None if narrow else p(enc.hist, np.int32), p(enc.movie_genre, np.int32),
                         p(enc.user_genre, np.int32), p(enc.numerics, np.float32),
                         p(enc.hist, np.uint16) if narrow else None)


class CTRModel:
    """One CTR ranking model resident on one GPU."""

    def __init__(self, spec: ModelSpec, weights: Mapping[str, object], device: int = 0,
                 narrow_ids: bool = False, options: Optional[Mapping[str, object]] = None):
        """`weights`: canonical name -> float32 numpy array (reference shapes), or a
        torch CUDA tensor for an embedding table that is already in HBM (used in
        place, see SRS_DEVICE_BORROWED in include/srs_ctr.h).  `narrow_ids`: host batches
        carry the history ids as uint16 (`srs_batch::hist16`, n_movies <= 65536).  A DIEN model may also
        be given the eight auxiliary-head tensors (`weights.aux_weight_shapes`) for `dien_outputs` /
        `dien_evaluate`.  `options`:
        kernel-variant choices for `srs_model_create_ex`, e.g. {"din_impl": "tc"}."""
        self.spec = spec
        self.narrow_ids = bool(narrow_ids) and spec.n_movies <= 65536
        self.device = int(device)
        self._h = None
        lib = _lib.load()
        self._lib = lib
        borrowed = {k for k, v in weights.items() if not isinstance(v, np.ndarray)}
        check_weights(spec, {k: v for k, v in weights.items() if k not in borrowed},
                      skip=tuple(borrowed))
        shapes = dict(weight_shapes(spec))
        self.has_aux = has_aux_weights(spec, weights)      # DIEN's optional auxiliary-head group
        if self.has_aux:
            shapes.update(aux_weight_shapes(spec))
        tensors = (_lib.SrsTensor * len(shapes))()
        self._keep = []
        for i, (name, shape) in enumerate(shapes.items()):
            if name not in weights:
                raise KeyError("missing weight tensor %r" % name)
            w = weights[name]
            rows = shape[0]
            cols = shape[1] if len(shape) > 1 else 1
            if name in borrowed:
                if tuple(w.shape) != tuple(shape) or str(w.dtype) != "torch.float32" or not w.is_contiguous():
                    raise ValueError("device tensor %r must be contiguous float32 %s" % (name, shape))
                self._keep.append(w)
                tensors[i] = _lib.SrsTensor(name.encode(), w.data_ptr(), rows, cols,
                                            _lib.SRS_DEVICE_BORROWED)
            else:
                a = np.ascontiguousarray(w, dtype=np.float32)
                self._keep.append(a)
                tensors[i] = _lib.SrsTensor(name.encode(), a.ctypes.data, rows, cols, _lib.SRS_HOST)
        handle = C.c_void_p()
        sp = _spec_struct(spec)
        opts = ";".join("%s=%s" % (k, v) for k, v in (options or {}).items()).encode()
        _lib.check(lib.srs_model_create_ex(C.byref(sp), tensors, len(shapes), self.device, opts or None,
                                           C.byref(handle)))
        self._h = handle
        self._keep = [w for w in self._keep if not isinstance(w, np.ndarray)]  # host copies done
        self.hist_cols = spec.hist_len if spec.model in ("din", "dien") \
            else (1 if spec.model == "widendeep" else 0)
        self.movie_table_rows = 0         # set_movie_table: the rows of the movie table in HBM

    # ---- constructors ------------------------------------------------------------
    @classmethod
    def from_spec(cls, spec: ModelSpec, seed: int = 0, device: int = 0, for_test: bool = True):
        return cls(spec, init_weights(spec, seed, for_test=for_test), device)

    @classmethod
    def from_savedmodel(cls, savedmodel_dir: str, model: str = "neuralcf", device: int = 0):
        """Load one of the reference's shipped exports (`webroot/modeldata/neuralcf/<v>`,
        `webroot/modeldata/MLPRec/005`) without TensorFlow."""
        from . import bundle
        if model == "neuralcf":
            return cls(default_spec("neuralcf"), bundle.load_neuralcf(savedmodel_dir), device)
        if model == "twotowers":
            return cls(default_spec("twotowers", hidden=(10,), final_dense=False),
                       bundle.load_twotowers(savedmodel_dir), device)
        raise ValueError("no shipped SavedModel layout known for %r" % model)

    # ---- lifetime ------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self._lib.srs_model_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def kernel_name(self) -> str:
        return self._lib.srs_model_kernel_name(self._h).decode()

    def set_sm_limit(self, n_sms: int):
        """At most `n_sms` CTAs per launch of the persistent tensor-core kernels (<= 0: all
        SMs), so that launches on other streams run beside it (`srs_model_set_sm_limit`)."""
        _lib.check(self._lib.srs_model_set_sm_limit(self._h, int(n_sms)))

    @property
    def bytes_per_inference(self) -> int:
        return int(self._lib.srs_model_bytes_per_inference(self._h))

    # ---- the reference's call surface -----------------------------------------------
    def predict(self, features: Mapping[str, object], batch_size: Optional[int] = None) -> np.ndarray:
        """`model.predict(x)`: feature dict of 1-D columns -> float32 [N,1]."""
        return self._predict(features, batch_size, want_logits=False)[0]

    def predict_with_logits(self, features, batch_size: Optional[int] = None):
        return self._predict(features, batch_size, want_logits=True)

    def _predict(self, features, batch_size, want_logits):
        enc = encode_batch(self.spec, features, narrow_ids=self.narrow_ids)
        n = enc.B
        probs = np.empty(n, np.float32)
        logits = np.empty(n, np.float32) if want_logits else None
        step = n if not batch_size else max(int(batch_size), 1)
        if n <= step:
            self.predict_encoded(enc, probs, logits)
        else:   # the Keras predict loop over dataset batches -> one pipelined library call
            bounds = [(lo, min(n, lo + step)) for lo in range(0, n, step)]
            self.predict_batches([enc.slice(lo, hi) for lo, hi in bounds],
                                 [probs[lo:hi] for lo, hi in bounds],
                                 None if logits is None else [logits[lo:hi] for lo, hi in bounds])
        return probs.reshape(n, 1), (None if logits is None else logits.reshape(n, 1))

    def predict_batches(self, encs, probs_list, logits_list=None):
        """`srs_predict_host_batches`: score a list of encoded batches, H2D / kernel / D2H of
        successive batches overlapped over the library's slots."""
        n = len(encs)
        keep = []
        structs = (_lib.SrsBatch * n)(*[_host_struct(e, keep) for e in encs])
        pp = (C.c_void_p * n)(*[p.ctypes.data for p in probs_list])
        lp = None
        if logits_list is not None:
            lp = (C.c_void_p * n)(*[l.ctypes.data for l in logits_list])
        _lib.check(self._lib.srs_predict_host_batches(self._h, n, structs, pp, lp))

    def predict_encoded(self, enc: EncodedBatch, probs: np.ndarray,
                        logits: Optional[np.ndarray] = None) -> np.ndarray:
        """Host arrays in, host scores out (`srs_predict_host`)."""
        if enc.B == 0:
            return probs
        keep = []
        b = _host_struct(enc, keep)
        assert probs.dtype == np.float32 and probs.flags.c_contiguous and probs.shape[0] == enc.B
        lp = None
        if logits is not None:
            assert logits.dtype == np.float32 and logits.flags.c_contiguous
            lp = logits.ctypes.data
        _lib.check(self._lib.srs_predict_host(self._h, C.byref(b), probs.ctypes.data, lp))
        return probs

    def rank(self, features: Mapping[str, object], size: int):
        """`RecForYouProcess.getRecList`'s tail for one request: score the candidate rows
        and return the best `size` (positions int32 [k], scores float32 [k], best first;
        equal scores by position) - `srs_rank_host`, only k results leave the device."""
        enc = encode_batch(self.spec, features, narrow_ids=self.narrow_ids)
        k = max(0, min(int(size), enc.B))
        idx = np.empty(k, np.int32)
        top = np.empty(k, np.float32)
        if k == 0:
            return idx, top
        keep = []
        b = _host_struct(enc, keep)
        _lib.check(self._lib.srs_rank_host(self._h, C.byref(b), k, idx.ctypes.data,
                                           top.ctypes.data))
        return idx, top

    def evaluate(self, features: Mapping[str, object], labels=None, batch_size: Optional[int] = None,
                 sample_weight=None):
        """`model.evaluate(x)` of a model compiled as every reference script compiles it
        (loss='binary_crossentropy', metrics=['accuracy', AUC(curve='ROC'), AUC(curve='PR')]):
        returns (loss, accuracy, roc_auc, pr_auc), Keras's order.  `labels` defaults to
        `features["label"]` (KeyError if missing); they must be 0 or 1.  Batches of `batch_size` rows
        (default: one) are scored and folded into the metrics on the device
        (`srs_evaluate_host_batches`); no score comes back.  ValueError for an out-of-range id, a bad
        label, a NaN or out-of-range probability, no rows, and the models evaluate does not cover
        (DIEN; two towers without the final Dense).  `sample_weight` ([N], Keras's `evaluate(...,
        sample_weight=)`) gives the weighted metrics of DESIGN.md section 4.28; ValueError for a weight that is
        negative, NaN or infinite or a length other than N (`training.sample_weights`)."""
        r = self.evaluate_result(features, labels, batch_size, sample_weight)
        return r.loss, r.accuracy, r.roc_auc, r.pr_auc

    def evaluate_result(self, features, labels=None, batch_size: Optional[int] = None,
                        sample_weight=None) -> _lib.SrsEvalResult:
        """`evaluate` with the counts: the `srs_eval_result` (rows, positives, correct and the four metrics)."""
        from .training import sample_weights
        lab = _label_array(features, labels)
        w = sample_weights(lab, sample_weight)
        enc = encode_batch(self.spec, features, narrow_ids=self.narrow_ids)
        n = enc.B
        if lab.shape[0] != n:
            raise ValueError("labels have %d rows, the features %d" % (lab.shape[0], n))
        if n == 0:
            raise ValueError("evaluate needs at least one row")
        step = n if not batch_size else max(int(batch_size), 1)
        bounds = [(lo, min(n, lo + step)) for lo in range(0, n, step)]
        keep = []
        structs = (_lib.SrsBatch * len(bounds))(*[_host_struct(enc.slice(lo, hi), keep) for lo, hi in bounds])
        lp = (C.c_void_p * len(bounds))(*[lab[lo:hi].ctypes.data for lo, hi in bounds])
        out = _lib.SrsEvalResult()
        if w is None:
            _lib.check(self._lib.srs_evaluate_host_batches(self._h, len(bounds), structs, lp, C.byref(out)))
            return out
        wp = (C.c_void_p * len(bounds))(*[w[lo:hi].ctypes.data for lo, hi in bounds])
        _lib.check(self._lib.srs_evaluate_weighted_host_batches(self._h, len(bounds), structs, lp, wp, C.byref(out)))
        return out

    # ---- DIEN's second output (DIEN.py:261-296) ---------------------------------------------------
    def _dien_batches(self, features, batch_size):
        """The Keras batches of a DIEN two-output call: (encoded batch, negatives, labels) structs and bounds."""
        lab = _label_array(features, None)
        if not np.all((lab == 0) | (lab == 1)):
            raise ValueError("labels must be 0 or 1")
        enc = encode_batch(self.spec, features, narrow_ids=self.narrow_ids)
        n = enc.B
        if lab.shape[0] != n:
            raise ValueError("labels have %d rows, the features %d" % (lab.shape[0], n))
        keys = negative_history_keys(self.spec.hist_len)
        neg = np.empty((n, max(len(keys), 1)), np.int32)
        for j, k in enumerate(keys):          # numeric_column ids like the history (DIEN.py:123-128), range-checked
            neg[:, j] = _as_ids(features, k, self.spec.n_movies, "negative movie id")
        neg = np.ascontiguousarray(neg[:, :len(keys)])
        step = n if not batch_size else max(int(batch_size), 1)
        bounds = [(lo, min(n, lo + step)) for lo in range(0, n, step)]
        keep = [neg, lab]
        structs = (_lib.SrsBatch * len(bounds))(*[_host_struct(enc.slice(lo, hi), keep) for lo, hi in bounds])
        negs = [np.ascontiguousarray(neg[lo:hi]) for lo, hi in bounds]
        keep += negs
        np_ = (C.c_void_p * len(bounds))(*[a.ctypes.data if a.size else None for a in negs])
        lp = (C.c_void_p * len(bounds))(*[lab[lo:hi].ctypes.data for lo, hi in bounds])
        return n, bounds, structs, np_, lp, keep

    def dien_outputs(self, features, batch_size: Optional[int] = None):
        """`model.predict(x)` of the reference's two-output DIEN (DIEN.py:296,312): `[y_pred float32 [N,1],
        final_loss float32 [N]]`.  `features` also carries `negtive_userRatedMovie2..T` (e.g. from
        `features.negative_history`) and `label` (0 or 1); a missing one raises KeyError, as Keras does for a
        missing input.  final_loss_i = bce_i - 0.5 * mean_j aux_j over the Keras batch of row i (DIEN.py:287),
        so it depends on `batch_size` (None: one batch).  y_pred has the bits of `predict`.  Needs the
        auxiliary-head weights (ValueError otherwise)."""
        n, bounds, structs, negs, lp, keep = self._dien_batches(features, batch_size)
        probs = np.empty(n, np.float32)
        final = np.empty(n, np.float32)
        pp = (C.c_void_p * len(bounds))(*[probs[lo:hi].ctypes.data for lo, hi in bounds])
        fp = (C.c_void_p * len(bounds))(*[final[lo:hi].ctypes.data for lo, hi in bounds])
        _lib.check(self._lib.srs_dien_outputs_host_batches(self._h, len(bounds), structs, negs, lp, pp, fp))
        return [probs.reshape(n, 1), final]

    def dien_evaluate(self, features, batch_size: Optional[int] = None) -> dict:
        """`model.evaluate(x, return_dict=True)` of the reference's DIEN (DIEN.py:298-304): {"loss", "auc",
        "auc_value"}, with Keras >= 2.3 semantics - the model is compiled without a loss or metrics, so Keras
        reports the `add_loss` value and the layer's own metrics:
          loss       the compile-less loss Mean over every element of each batch's final_loss: the sum over all
                     rows / N;
          auc        the layer's `tf.keras.metrics.AUC()` over all (label, y_pred) (200 thresholds, exact counts;
                     the roc_auc of `evaluate`);
          auc_value  `add_metric(self.auc.result(), aggregation="mean")`: the mean over batches k of the AUC of
                     batches 0..k, so it depends on the batch order.
        Keras >= 2.3 because DIEN.py:41-42 drops the last partial batch only for TF < 2.3, whose loss is aggregated
        per batch position; this keeps every row.  Batches of `batch_size` rows (None: one batch).  Inputs and
        errors as `dien_outputs`."""
        n, bounds, structs, negs, lp, keep = self._dien_batches(features, batch_size)
        if n == 0:
            raise ValueError("evaluate needs at least one row")
        out = _lib.SrsDienEvalResult()
        _lib.check(self._lib.srs_dien_evaluate_host_batches(self._h, len(bounds), structs, negs, lp, C.byref(out)))
        return {"loss": out.loss, "auc": out.auc, "auc_value": out.auc_value}

    # ---- one user x n candidates, movie features resident in HBM ----------------------------
    def set_movie_table(self, table):
        """Upload the movie side of the serving feature store (`featurestore.MovieFeatureTable`,
        i.e. the `mf:<movieId>` hashes of FeatureEngForRecModel.scala:130-174) to HBM once;
        `rank_user` requests then carry only the user's row and the candidate ids."""
        n = table.n_movies
        genres = np.ascontiguousarray(np.stack([table.idx_cols[k] for k in
                                                ("movieGenre1", "movieGenre2", "movieGenre3")], axis=1), np.int32)
        nums = np.ascontiguousarray(np.stack([
            table.float_cols["movieAvgRating"], table.int_cols["movieRatingCount"].astype(np.float32),
            table.float_cols["movieRatingStddev"], table.int_cols["releaseYear"].astype(np.float32)], axis=1),
            np.float32)
        _lib.check(self._lib.srs_model_set_movie_features(self._h, n, genres.ctypes.data, nums.ctypes.data))
        self.movie_table_rows = n

    def rank_user(self, user_id: int, user_fields: Mapping[str, object], candidate_ids, size: int,
                  return_scores: bool = False):
        """`RecForYouProcess.getRecList` for one request (`:40-59`): `user_fields` is the user's
        `uf:` hash (strings, as `FeatureStore.user_features` returns it, or already typed values
        under the model input names), `candidate_ids` the n candidate movies.  Ships the user's
        row and the ids only (`srs_rank_user_host`); the movie features are gathered on the
        device from the table uploaded by `set_movie_table`.  Returns (positions int32 [k],
        scores float32 [k]) best first (+ all n scores with `return_scores`)."""
        from .featurestore import parse_user_features
        from .features import genre_to_index
        typed = parse_user_features(user_fields, max(self.hist_cols, 1))
        cand = np.ascontiguousarray(np.asarray(candidate_ids, np.int32).reshape(-1))
        n = cand.shape[0]
        k = max(0, min(int(size), n))
        from .spec import history_keys
        hkeys = history_keys(self.spec.hist_len) if self.spec.model in ("din", "dien") else ["userRatedMovie1"]
        hist = np.ascontiguousarray(np.array([typed[k] for k in hkeys[:self.hist_cols]], np.int32))   # graph position order
        row = _lib.SrsUserRow()
        row.user_id = int(user_id)
        for g in range(5):
            v = typed["userGenre%d" % (g + 1)]
            row.user_genre[g] = int(genre_to_index([v])[0]) if isinstance(v, (str, bytes)) else int(v)
        row.user_numerics[0] = float(typed["userAvgRating"])
        row.user_numerics[1] = float(np.float32(typed["userRatingCount"]))
        row.user_numerics[2] = float(typed["userRatingStddev"])
        row.n_hist = self.hist_cols
        row.hist = hist.ctypes.data if self.hist_cols else None
        idx = np.empty(k, np.int32)
        top = np.empty(k, np.float32)
        probs = np.empty(n, np.float32) if return_scores else None
        _lib.check(self._lib.srs_rank_user_host(self._h, C.byref(row), cand.ctypes.data, n, k,
                                                idx.ctypes.data if k else None, top.ctypes.data if k else None,
                                                probs.ctypes.data if return_scores else None))
        return (idx, top, probs) if return_scores else (idx, top)

    # ---- pipelined host path -----------------------------------------------------------
    def num_slots(self) -> int:
        return int(self._lib.srs_num_slots())

    def submit_host(self, slot: int, batch_struct: _lib.SrsBatch, probs_ptr: int,
                    logits_ptr: Optional[int] = None):
        _lib.check(self._lib.srs_predict_host_async(self._h, slot, C.byref(batch_struct),
                                                    probs_ptr, logits_ptr))

    def wait(self, slot: int):
        _lib.check(self._lib.srs_wait_slot(self._h, slot))

    # ---- device-resident path -----------------------------------------------------------
    def to_device(self, features_or_enc) -> DeviceBatch:
        enc = features_or_enc if isinstance(features_or_enc, EncodedBatch) \
            else encode_batch(self.spec, features_or_enc)
        return DeviceBatch(enc, "cuda:%d" % self.device, self.hist_cols)

    def predict_device(self, batch: DeviceBatch, probs, logits=None, stream=None):
        """Everything in HBM: `probs` / `logits` are float32 CUDA tensors [B]; asynchronous
        on `stream` (a torch stream; default: torch's current stream)."""
        import torch
        if stream is None:
            stream = torch.cuda.current_stream(self.device)
        b = batch.struct()
        _lib.check(self._lib.srs_predict_device(
            self._h, C.byref(b), probs.data_ptr(), None if logits is None else logits.data_ptr(),
            stream.cuda_stream))
        return probs

    def status(self):
        """Synchronise; raises ValueError if a device batch carried an out-of-range id."""
        _lib.check(self._lib.srs_model_status(self._h))


class Metrics:
    """Keras's evaluate metrics accumulated on the device (`srs_metrics`): fold batches whose scores are
    already in HBM - e.g. straight after `CTRModel.predict_device`, in the same CUDA graph - and read
    the four numbers once at the end."""

    def __init__(self, device: int = 0):
        self._lib = _lib.load()
        self.device = int(device)
        self._h = None
        h = C.c_void_p()
        _lib.check(self._lib.srs_metrics_create(self.device, C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.srs_metrics_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _stream(self, stream):
        import torch
        return (stream if stream is not None else torch.cuda.current_stream(self.device)).cuda_stream

    def update_device(self, probs, logits, labels, stream=None, weights=None):
        """Fold n rows: `probs`, `logits` float32 and `labels` int32 CUDA tensors [n], asynchronous on
        `stream` (a torch stream; default: torch's current stream).  `weights` (float32 CUDA tensor [n]): Keras's
        sample weights (DESIGN.md section 4.28); a state folds either weighted or unweighted rows between resets."""
        n = int(probs.numel())
        cols = [("probs", probs, "torch.float32"), ("logits", logits, "torch.float32"), ("labels", labels, "torch.int32")]
        if weights is not None:
            cols.append(("weights", weights, "torch.float32"))
        for name, t, dt in cols:
            if str(t.dtype) != dt or not t.is_cuda or not t.is_contiguous() or int(t.numel()) != n:
                raise ValueError("%s must be a contiguous %s CUDA tensor of %d elements" % (name, dt[6:], n))
        if weights is None:
            _lib.check(self._lib.srs_metrics_update_device(self._h, probs.data_ptr(), logits.data_ptr(),
                                                           labels.data_ptr(), n, self._stream(stream)))
        else:
            _lib.check(self._lib.srs_metrics_update_weighted_device(self._h, probs.data_ptr(), logits.data_ptr(),
                                                                    labels.data_ptr(), weights.data_ptr(), n,
                                                                    self._stream(stream)))

    def reset(self, stream=None):
        _lib.check(self._lib.srs_metrics_reset(self._h, self._stream(stream)))

    def result(self) -> dict:
        """Synchronise and summarise: loss, accuracy, roc_auc, pr_auc, rows, positives, correct, and the
        confusion counts tp, fp, tn, fn (int64 [200] each, one per Keras threshold)."""
        out = _lib.SrsEvalResult()
        conf = np.zeros((4, 200), np.int64)
        _lib.check(self._lib.srs_metrics_result(self._h, C.byref(out), conf.ctypes.data))
        r = {k: getattr(out, k) for k, _ in _lib.SrsEvalResult._fields_}
        r.update(tp=conf[0], fp=conf[1], tn=conf[2], fn=conf[3])
        return r


def _label_array(features, labels=None) -> np.ndarray:
    """`labels` (default: `features["label"]`, KeyError if missing) as int32 [N]; ValueError unless integral."""
    if labels is None:
        if "label" not in features:
            raise KeyError("missing required feature 'label' (or pass labels=)")
        labels = features["label"]
    lab = np.asarray(labels)
    if lab.ndim == 2 and lab.shape[1] == 1:
        lab = lab[:, 0]
    if lab.ndim != 1:
        raise ValueError("labels must be 1-D [N], got shape %s" % (lab.shape,))
    if lab.dtype.kind == "f" and not np.all(lab == np.trunc(lab)):
        raise ValueError("labels must be 0 or 1")
    if lab.dtype.kind not in "biuf":
        raise ValueError("labels must be numeric 0 or 1")
    if lab.size and (lab.min() < np.iinfo(np.int32).min or lab.max() > np.iinfo(np.int32).max):
        raise ValueError("labels must be 0 or 1")
    return np.ascontiguousarray(lab, np.int32)            # the library rejects anything but 0 and 1


def launch_count() -> int:
    return int(_lib.load().srs_launch_count())
