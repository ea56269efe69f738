"""din_wg_kernel (csrc/din_wg.cu) runs as many warpgroups per CTA as its registers allow without spilling:
compile it for sm_90a with ptxas's resource report and hold both instantiations to zero spill bytes, so that
a later edit cannot trade the warpgroups' occupancy for local-memory traffic unnoticed.  No GPU needed."""
import os
import re
import subprocess
import tempfile

from sparrowrecsys_b200 import build


def test_din_wg_kernel_compiles_spill_free():
    src = os.path.join(build.CSRC, "din_wg.cu")
    with tempfile.TemporaryDirectory(prefix="srs_din_wg_res_") as tmp:
        cmd = [build.nvcc_path(), *build.ARCH, "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
               "--extended-lambda", "-Xptxas", "-v", "-c", src, "-o", os.path.join(tmp, "din_wg.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out
    # ptxas prints, per entry function: "Compiling entry function '<name>'", then "N bytes stack frame,
    # S bytes spill stores, L bytes spill loads" and "Used R registers"
    blocks = re.split(r"Compiling entry function '", out)[1:]
    found = {}
    for blk in blocks:
        name = blk.split("'", 1)[0]
        m = re.search(r"din_wg_kernelILi(\d+)E", name)
        if not m:
            continue
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", blk)
        assert spill, blk
        found[int(m.group(1))] = (int(spill.group(1)), int(spill.group(2)))
    assert sorted(found) == [32, 64], out
    for ep, (st, ld) in found.items():
        assert st == 0 and ld == 0, "din_wg_kernel<%d> spills: %d bytes stored, %d loaded" % (ep, st, ld)
