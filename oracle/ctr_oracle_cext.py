"""ctypes loader for oracle/ctr_oracle_c.c - the plain-C, OpenMP-threaded restatement of the
reference's DIN graph used as the CPU *timing* baseline (bench.py cpu_baseline / --impl
reference) and cross-checked against the numpy oracle in tests/test_oracle_c.py.

THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT (see ctr_oracle.py).  Feature-column
handling (vocabulary lookup of genre strings, float32 round trip of the DIN ids, range asserts)
is done here with the numpy oracle's own primitives, then the encoded arrays go to C.

Build: `python -m oracle.ctr_oracle_cext` (or __graft_entry__.build()) ->
oracle/libctr_oracle_c.so, compiled with gcc -O3 -mavx2 -mfma -fopenmp (a generic -O3 build
is kept next to it for hosts without AVX2).  The .so files are build products, like the product
library, and are not tracked by git."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from . import ctr_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "ctr_oracle_c.c")
LIB_AVX2 = os.path.join(HERE, "libctr_oracle_c.so")
LIB_GENERIC = os.path.join(HERE, "libctr_oracle_c_generic.so")


def build(force: bool = False):
    gcc = shutil.which("gcc") or "/usr/bin/gcc"
    out = []
    for lib, flags in ((LIB_AVX2, ["-mavx2", "-mfma"]), (LIB_GENERIC, [])):
        if force or not os.path.exists(lib) or os.path.getmtime(lib) < os.path.getmtime(SRC):
            subprocess.check_call([gcc, "-O3", "-fopenmp", "-shared", "-fPIC", "-std=c11", *flags,
                                   "-o", lib, SRC, "-lm"])
        out.append(lib)
    return out


def _host_has_avx2() -> bool:
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    fl = line.split()
                    return "avx2" in fl and "fma" in fl
    except OSError:
        pass
    return False


class _Din(C.Structure):
    _fields_ = [("T", C.c_int32), ("E", C.c_int32), ("AU", C.c_int32), ("H1", C.c_int32), ("H2", C.c_int32),
                ("n_movies", C.c_int32), ("n_users", C.c_int32), ("n_genres", C.c_int32),
                ("emb", C.c_void_p), ("user_emb", C.c_void_p), ("ugenre_emb", C.c_void_p),
                ("mgenre_emb", C.c_void_p), ("au_w", C.c_void_p), ("au_b", C.c_void_p),
                ("au_alpha", C.c_void_p), ("au_out_w", C.c_void_p), ("au_out_b", C.c_float),
                ("w1", C.c_void_p), ("b1", C.c_void_p), ("a1", C.c_void_p), ("w2", C.c_void_p),
                ("b2", C.c_void_p), ("a2", C.c_void_p), ("w3", C.c_void_p), ("b3", C.c_float)]


_lib = None


def load():
    global _lib
    if _lib is None:
        # idle OpenMP workers sleep instead of spinning: a thread-count sweep otherwise leaves the workers of
        # the larger teams spinning on the cores the next measurement needs (seen as 25x swings on a 128-CPU host)
        os.environ.setdefault("OMP_WAIT_POLICY", "PASSIVE")
        os.environ.setdefault("GOMP_SPINCOUNT", "0")
        os.environ.setdefault("OMP_PROC_BIND", "false")
        os.environ.setdefault("OMP_DYNAMIC", "false")
        path = LIB_AVX2 if _host_has_avx2() else LIB_GENERIC
        if not os.path.exists(path):
            build()
        lib = C.CDLL(path)
        lib.srs_oracle_din_forward.restype = C.c_int
        lib.srs_oracle_din_forward.argtypes = [C.POINTER(_Din), C.c_int32] + [C.c_void_p] * 3 + [C.c_int32] + \
            [C.c_void_p] * 5 + [C.c_int32]
        lib.srs_oracle_max_threads.restype = C.c_int
        _lib = lib
    return _lib


def encode_din(spec, feats):
    """Feature dict -> the encoded arrays (what the feature columns of DIN.py:95-123 produce)."""
    keys = O.din_history_keys(spec.hist_len)
    f32ids = lambda k: np.asarray(feats[k]).astype(np.float32).astype(np.int32)      # :95,125 float round trip
    movie = np.ascontiguousarray(f32ids("movieId"))
    hist = np.ascontiguousarray(np.stack([f32ids(k) for k in keys], axis=1))
    user = np.ascontiguousarray(O.identity_ids(feats, "userId", spec.n_users).astype(np.int32))
    ug = np.ascontiguousarray(O.genre_index(feats, "userGenre1").astype(np.int32))
    mg = np.ascontiguousarray(O.genre_index(feats, "movieGenre1").astype(np.int32))
    nk = ("movieAvgRating", "movieRatingCount", "movieRatingStddev", "releaseYear", "userAvgRating",
          "userRatingCount", "userRatingStddev")
    nums = np.ascontiguousarray(np.stack([np.asarray(feats[k]).astype(np.float32) for k in nk], axis=1))
    return movie, user, hist, ug, mg, nums


def din_predictor(spec, W, threads=None):
    """forward(feats) -> (prob [B,1], logit [B,1]) through the C restatement on `threads` OpenMP
    threads; forward.encoded(arrays) skips the feature-column step (for timing the graph alone)."""
    lib = load()
    threads = int(threads or os.cpu_count() or 1)
    keep = {k: np.ascontiguousarray(np.asarray(v), np.float32) for k, v in W.items()}
    p = lambda k: keep[k].ctypes.data
    m = _Din(spec.hist_len, spec.emb_dim, spec.au_hidden, spec.hidden[0], spec.hidden[1],
             spec.n_movies, spec.n_users, spec.n_genres,
             p("embedding"), p("userId_embedding"), p("userGenre1_embedding"), p("movieGenre1_embedding"),
             p("au_dense/kernel"), p("au_dense/bias"), p("au_prelu/alpha"), p("au_out/kernel"),
             float(keep["au_out/bias"].reshape(-1)[0]),
             p("dense/kernel"), p("dense/bias"), p("prelu/alpha"), p("dense_1/kernel"), p("dense_1/bias"),
             p("prelu_1/alpha"), p("dense_2/kernel"), float(keep["dense_2/bias"].reshape(-1)[0]))

    def encoded(arrs, nthreads=None):
        movie, user, hist, ug, mg, nums = arrs
        B = movie.shape[0]
        prob = np.empty((B, 1), np.float32)
        logit = np.empty((B, 1), np.float32)
        rc = lib.srs_oracle_din_forward(C.byref(m), B, movie.ctypes.data, user.ctypes.data, hist.ctypes.data,
                                        hist.shape[1], ug.ctypes.data, mg.ctypes.data, nums.ctypes.data,
                                        prob.ctypes.data, logit.ctypes.data, int(nthreads or threads))
        if rc != 0:
            raise ValueError("movie/user id out of range")
        return prob, logit

    def forward(feats, nthreads=None):
        return encoded(encode_din(spec, feats), nthreads)

    forward.encoded = encoded
    forward.keep = (keep, m)
    return forward


if __name__ == "__main__":
    print(build(force=True))
