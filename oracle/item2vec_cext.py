"""ctypes loader for oracle/item2vec_c.c - oracle/item2vec.py's training loop in plain C, for full runs and as the
CPU timing baseline of tools/item2vec_throughput.py.

THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Build: `python -m oracle.item2vec_cext` (or
__graft_entry__.build()) -> oracle/libitem2vec_c.so, compiled with -ffp-contract=off so that no multiply-add is
fused; the .so is a build product and is not tracked by git."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from . import item2vec as I

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "item2vec_c.c")
LIB = os.path.join(HERE, "libitem2vec_c.so")

_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        gcc = shutil.which("gcc") or "/usr/bin/gcc"
        tmp = LIB + ".tmp%d" % os.getpid()
        subprocess.check_call([gcc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-std=c11",
                               "-o", tmp, SRC])
        os.replace(tmp, LIB)
    return LIB


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        lib = C.CDLL(LIB)
        lib.srs_oracle_item2vec_train.restype = C.c_int
        lib.srs_oracle_item2vec_train.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                                  C.c_int32, C.c_int32, C.c_uint64, C.c_int64, C.c_double,
                                                  C.c_void_p]
        _lib = lib
    return _lib


def train(words, offs, counts, code, point, codelen, vector_size, window, iterations, partitions, seed,
          lr=I.LEARNING_RATE):
    """oracle/item2vec.py's `train` in C: returns syn0 [V][vector_size] float32."""
    V = len(counts)
    syn0 = np.ascontiguousarray(I.init_syn0(seed, V, vector_size))
    a = [np.ascontiguousarray(x, t) for x, t in ((words, np.int32), (offs, np.int64), (code, np.int8),
                                                 (point, np.int32), (codelen, np.int32),
                                                 (I.exp_table(), np.float32))]
    rc = load().srs_oracle_item2vec_train(a[0].ctypes.data, a[1].ctypes.data, len(offs) - 1, a[2].ctypes.data,
                                          a[3].ctypes.data, a[4].ctypes.data, a[5].ctypes.data, V, vector_size,
                                          window, iterations, partitions, seed & ((1 << 64) - 1),
                                          int(np.sum(counts)), lr, syn0.ctypes.data)
    if rc != 0:
        raise MemoryError("item2vec oracle: out of memory")
    return syn0


def item2vec(user, movie, half, ts, vector_size=10, window=5, iterations=10, partitions=1, seed=0):
    """ratings -> (vocabulary ids [V], vectors [V][vector_size]), the training loop in C."""
    _, seqs = I.positive_sequences(user, movie, half, ts)
    ids, counts = I.build_vocab(seqs)
    words, offs = I.chunk_corpus(seqs, ids)
    code, point, codelen = I.huffman(counts)
    return ids, train(words, offs, counts, code, point, codelen, vector_size, window, iterations, partitions, seed)


if __name__ == "__main__":
    print(build(force=True))
