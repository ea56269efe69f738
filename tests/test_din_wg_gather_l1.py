"""din_wg_kernel copies its gathered embedding rows through L1 (cp.async.ca), not around it (cp.async.cg, SASS
LDGSTS.E.BYPASS): a few rows (the padding row, popular movies, the 20 genre rows) are read again and again, and
an SM that has read one finds it in its L1 instead of queueing on one L2 line with every other SM.  Compile
din_wg.cu for sm_90a and read the SASS of both instantiations: every 16-byte copy with a zero-fill operand (the
history, candidate and side-feature rows, whose source size is 0 past a row's length or for a missing row)
must be the L1-cached form.  The staged weights, read once per CTA, are copied without a zero fill and may
bypass L1.  No GPU needed."""
import os
import re
import subprocess
import tempfile

from sparrowrecsys_b200 import build

# "LDGSTS.E.BYPASS.128 [R7], desc[UR6][R2.64], P0 ;": the trailing predicate (or a .ZFILL suffix) is the
# zero fill of a copy with a source size
LDGSTS = re.compile(r"LDGSTS(?P<mods>(\.[A-Z0-9]+)*)\s+\[[^\]]*\],\s*(desc\[[^\]]*\])?\[[^\]]*\](?P<zf>,\s*!?P\d)?\s*;")


def sass(src):
    cuobjdump = os.path.join(os.path.dirname(build.nvcc_path()), "cuobjdump")
    with tempfile.TemporaryDirectory(prefix="srs_gather_l1_") as tmp:
        cubin = os.path.join(tmp, "k.cubin")
        cmd = [build.nvcc_path(), *build.ARCH, "-O3", "-std=c++17", "--expt-relaxed-constexpr",
               "--extended-lambda", "-cubin", os.path.join(build.CSRC, src), "-o", cubin]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        r = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def test_din_wg_row_gathers_go_through_l1():
    seen = []
    for f in re.split(r"\n\s*Function : ", sass("din_wg.cu"))[1:]:
        name = f.split("\n", 1)[0].strip()
        m = re.search(r"din_wg_kernelILi(\d+)E", name)
        if not m:
            continue
        seen.append(int(m.group(1)))
        copies = [c for c in LDGSTS.finditer(f) if ".128" in c.group("mods")]
        gathers = [c for c in copies if c.group("zf") or ".ZFILL" in c.group("mods")]
        assert gathers, "%s: no zero-filling 16-byte LDGSTS" % name
        bypass = [c.group(0) for c in gathers if ".BYPASS" in c.group("mods")]
        assert not bypass, "%s: %d of %d row gathers bypass L1, e.g. %s" % (name, len(bypass), len(gathers),
                                                                            bypass[0])
    assert sorted(seen) == [32, 64], seen
