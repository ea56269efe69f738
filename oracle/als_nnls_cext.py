"""ctypes loader for oracle/als_nnls_c.c - oracle/als_nnls.py's nonnegative ALS half-step in plain C, for full runs
and as the CPU timing baseline of tools/als_nonnegative_throughput.py.

THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Build: `python -m oracle.als_nnls_cext` (or
__graft_entry__.build()) -> oracle/libals_nnls_c.so, compiled with -ffp-contract=off so that no multiply-add is
fused; the .so is a build product and is not tracked by git.  The init and YtY come from oracle/als_c.c and
oracle/als_implicit_c.c."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from . import als_cext as X
from . import als_implicit_cext as XI
from . import als_nnls as N

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "als_nnls_c.c")
LIB = os.path.join(HERE, "libals_nnls_c.so")

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
        lib.srs_oracle_als_solve_nnls.restype = I32
        lib.srs_oracle_als_solve_nnls.argtypes = [V, V, V, I32, V, V, V, I32, F64, F64, V]
        _lib = lib
    return _lib


def _p(a):
    return a.ctypes.data


def solve_half(lay, srcF, src_ids, k, reg, alpha=None, iters=None):
    """oracle/als_nnls.solve_half in C; `iters`, an int32 [nE] array, receives each entity's NNLS iterations."""
    off, src, r = (np.ascontiguousarray(x, t) for x, t in zip(lay, (np.int32, np.int32, np.float32)))
    srcF = np.ascontiguousarray(srcF, np.float32)
    yty = None if alpha is None else np.ascontiguousarray(XI.yty(src_ids, srcF))
    out = np.zeros((len(off) - 1, k), np.float32)
    if load().srs_oracle_als_solve_nnls(_p(off), _p(src), _p(r), len(off) - 1, _p(srcF),
                                        None if yty is None else _p(yty), _p(out), k, float(reg),
                                        0.0 if alpha is None else float(alpha),
                                        None if iters is None else _p(iters)) == -2:
        raise MemoryError("ALS oracle: out of memory")
    return out, -1


def fit(user, movie, rating, rank=10, max_iter=5, reg_param=0.01, seed=0, implicit_prefs=False, alpha=1.0,
        solver=solve_half):
    """oracle/als_nnls.py's `fit`, each half-step in C."""
    return N.fit(user, movie, rating, rank, max_iter, reg_param, seed, implicit_prefs, alpha, solver=solver,
                 init=X.init_user_factors)


if __name__ == "__main__":
    print(build(force=True))
