"""Build the CUDA library in-tree: `python -m sparrowrecsys_b200.build`.

nvcc cross-compiles for sm_90a (H100) without a GPU; the resulting
`sparrowrecsys_b200/libsrs_ctr.so` is a build product and is not tracked by git.
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsrs_ctr.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def headers():
    """Everything every object depends on besides its own source: the headers, and this file, which
    holds the architecture and compiler flags."""
    return glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh")) \
        + glob.glob(os.path.join(os.path.dirname(HERE), "include", "*.h")) + [os.path.abspath(__file__)]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in sources() + headers())


def build(force: bool = False, verbose: bool = False, defines=(), out_dir: str = None) -> str:
    """Compile and link the library; returns its path.  `defines` (e.g. ["SRS_DIN_PHASES"]) build a
    variant, which needs `out_dir`: its objects and library go there, never over the in-tree build."""
    if defines and not out_dir:
        raise ValueError("a build with extra defines needs its own out_dir")
    lib = os.path.join(out_dir, "libsrs_ctr.so") if out_dir else LIB
    if not out_dir and not force and not needs_build():
        return LIB
    objdir = os.path.join(out_dir or os.path.join(HERE, "build"), ARCH[1].split("code=")[1])   # objects of another arch never mix in
    os.makedirs(objdir, exist_ok=True)
    nvcc = nvcc_path()
    common = [nvcc, *ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr", "--extended-lambda"] + ["-D" + d for d in defines]
    if verbose:
        common += ["-Xptxas", "-v"]
    procs = []
    objs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if (not force and os.path.exists(obj)
                and os.path.getmtime(obj) > max(os.path.getmtime(d) for d in [src] + headers())):
            continue
        procs.append((src, subprocess.Popen(common + ["-c", src, "-o", obj],
                                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = False
    for src, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed on %s:\n%s\n" % (src, out))
        elif verbose or out.strip():
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("CUDA build failed")
    tmp = lib + ".tmp%d" % os.getpid()                   # link aside, then rename: a reader (or a copy of
    subprocess.check_call([nvcc, *ARCH, "-shared", "-o", tmp, *objs])   # the tree) never sees a half-written library
    os.replace(tmp, lib)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
