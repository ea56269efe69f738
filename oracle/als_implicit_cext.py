"""ctypes loader for oracle/als_implicit_c.c - oracle/als_implicit.py's implicit ALS half-step, YtY and
RankingMetrics in plain C, for full runs and as the CPU timing baseline of tools/als_implicit_throughput.py.

THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Build: `python -m oracle.als_implicit_cext` (or
__graft_entry__.build()) -> oracle/libals_implicit_c.so, compiled with -ffp-contract=off so that no multiply-add is
fused; the .so is a build product and is not tracked by git."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from . import als_cext as X
from . import als_implicit as I

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "als_implicit_c.c")
LIB = os.path.join(HERE, "libals_implicit_c.so")

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
        V, I32, F64 = C.c_void_p, C.c_int32, C.c_double
        lib.srs_oracle_als_yty.restype = I32
        lib.srs_oracle_als_yty.argtypes = [V, I32, V, I32, V, V]
        lib.srs_oracle_als_solve_implicit.restype = I32
        lib.srs_oracle_als_solve_implicit.argtypes = [V, V, V, I32, V, V, I32, V, I32, F64, F64]
        lib.srs_oracle_ranking_metrics.restype = I32
        lib.srs_oracle_ranking_metrics.argtypes = [V, I32, I32, V, V, I32, V, V]
        _lib = lib
    return _lib


def _p(a):
    return a.ctypes.data


def yty(ids, srcF, order=tuple(range(I.BLOCKS))):
    """Packed YtY [k (k + 1) / 2] (see oracle/als_implicit.yty)."""
    ids = np.ascontiguousarray(ids, np.int32)
    srcF = np.ascontiguousarray(srcF, np.float32)
    k = srcF.shape[1]
    ordr = np.ascontiguousarray(order, np.int32)
    out = np.zeros(k * (k + 1) // 2)
    if load().srs_oracle_als_yty(_p(ids), len(ids), _p(srcF), k, _p(ordr), _p(out)) == -2:
        raise MemoryError("ALS oracle: out of memory")
    return out


def solve_half(lay, srcF, src_ids, k, reg, alpha):
    off, src, r = (np.ascontiguousarray(x, t) for x, t in zip(lay, (np.int32, np.int32, np.float32)))
    srcF = np.ascontiguousarray(srcF, np.float32)
    ids = np.ascontiguousarray(src_ids, np.int32)
    out = np.zeros((len(off) - 1, k), np.float32)
    bad = load().srs_oracle_als_solve_implicit(_p(off), _p(src), _p(r), len(off) - 1, _p(srcF), _p(ids), len(ids),
                                               _p(out), k, float(reg), float(alpha))
    if bad == -2:
        raise MemoryError("ALS oracle: out of memory")
    return out, int(bad)


def fit(user, movie, rating, rank=10, max_iter=5, reg_param=0.01, alpha=1.0, seed=0):
    """oracle/als_implicit.py's `fit`, each half-step in C."""
    return I.fit(user, movie, rating, rank, max_iter, reg_param, alpha, seed, solver=solve_half,
                 init=X.init_user_factors)


def ranking_metrics(pred_ids, label_off, label_ids, k):
    """(means [3], per-query [3][n]) from pred_ids [n][L] and labels in CSR form."""
    pred = np.ascontiguousarray(pred_ids, np.int32)
    off = np.ascontiguousarray(label_off, np.int32)
    lab = np.ascontiguousarray(label_ids, np.int32)
    n = len(off) - 1
    L = pred.shape[1] if pred.ndim == 2 else 0
    out = np.zeros((3, n))
    means = np.zeros(3)
    if load().srs_oracle_ranking_metrics(_p(pred), n, L, _p(off), _p(lab if lab.size else np.zeros(1, np.int32)),
                                         int(k), _p(out), _p(means)) == -2:
        raise MemoryError("ranking oracle: out of memory")
    return means, out


if __name__ == "__main__":
    print(build(force=True))
