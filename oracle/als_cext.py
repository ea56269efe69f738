"""ctypes loader for oracle/als_c.c - oracle/als.py's ALS and recommendForAll in plain C, for full runs and as the
CPU timing baseline of tools/als_throughput.py.

THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Build: `python -m oracle.als_cext` (or
__graft_entry__.build()) -> oracle/libals_c.so, compiled with -ffp-contract=off so that no multiply-add is fused;
the .so is a build product and is not tracked by git."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from . import als as A

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "als_c.c")
LIB = os.path.join(HERE, "libals_c.so")

_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        gcc = shutil.which("gcc") or "/usr/bin/gcc"
        tmp = LIB + ".tmp%d" % os.getpid()
        subprocess.check_call([gcc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-std=c11",
                               "-o", tmp, SRC, "-lm"])
        os.replace(tmp, LIB)
    return LIB


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        lib = C.CDLL(LIB)
        lib.srs_oracle_als_init.restype = None
        lib.srs_oracle_als_init.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_uint64, C.c_void_p]
        lib.srs_oracle_als_solve.restype = C.c_int32
        lib.srs_oracle_als_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_int32, C.c_double]
        lib.srs_oracle_als_recommend.restype = None
        lib.srs_oracle_als_recommend.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                                 C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib


def _p(a):
    return a.ctypes.data


def init_user_factors(user_ids, rank, seed):
    ids = np.ascontiguousarray(user_ids, np.int32)
    out = np.zeros((len(ids), rank), np.float32)
    load().srs_oracle_als_init(_p(ids), len(ids), rank, seed & ((1 << 64) - 1), _p(out))
    return out


def solve_half(lay, srcF, k, reg):
    off, src, r = (np.ascontiguousarray(x, t) for x, t in zip(lay, (np.int32, np.int32, np.float32)))
    srcF = np.ascontiguousarray(srcF, np.float32)
    out = np.zeros((len(off) - 1, k), np.float32)
    bad = load().srs_oracle_als_solve(_p(off), _p(src), _p(r), len(off) - 1, _p(srcF), _p(out), k, float(reg))
    if bad == -2:
        raise MemoryError("ALS oracle: out of memory")
    return out, int(bad)


def fit(user, movie, rating, rank=10, max_iter=5, reg_param=0.01, seed=0):
    """oracle/als.py's `fit`, each half-step in C."""
    return A.fit(user, movie, rating, rank, max_iter, reg_param, seed, solver=solve_half, init=init_user_factors)


def recommend(src, dst_ids, dst, num):
    src = np.ascontiguousarray(src, np.float32)
    dst = np.ascontiguousarray(dst, np.float32)
    ids = np.ascontiguousarray(dst_ids, np.int32)
    k = src.shape[1] if src.ndim == 2 else dst.shape[1]
    L = min(int(num), dst.shape[0])
    oi = np.zeros((src.shape[0], L), np.int32)
    os_ = np.zeros((src.shape[0], L), np.float32)
    load().srs_oracle_als_recommend(_p(src), src.shape[0], _p(ids), _p(dst), dst.shape[0], k, L, _p(oi), _p(os_))
    return oi, os_


if __name__ == "__main__":
    print(build(force=True))
