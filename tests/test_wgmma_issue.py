"""The wgmma conv kernel must issue each chunk's MMAs as one chained batch (checked in the SASS, no GPU needed).

ptxas serializes wgmma when a runtime condition guards one of them, or when the accumulator registers are touched
between them: it then fences every HGMMA with its own WARPGROUP.ARRIVE and waits for it (WARPGROUP.DEPBAR) before the
next one is issued, and the tensor pipe runs one dependent MMA at a time.  That costs up to 2x on the conv layers while
every result stays the same, so only the instruction stream shows it.
"""
import os
import re
import shutil
import subprocess

import pytest


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if c and os.path.exists(c):
            return c
    return None


def _kernels(sass):
    """{template arguments of conv_tc_kernel: [HGMMA, WARPGROUP.ARRIVE, WARPGROUP.DEPBAR] counts}."""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            t = re.search(r"conv_tc_kernelI((?:L[ib]n?\d+E)+)E", m.group(1))
            # Li1E = 1, Lin1E = -1, Lb0E = false
            cur = tuple(int(v) * (-1 if n else 1) for _, n, v in re.findall(r"L([ib])(n?)(\d+)E", t.group(1))) if t else None
            if cur is not None:
                out[cur] = [0, 0, 0]
            continue
        if cur is None:
            continue
        if "HGMMA" in line:
            out[cur][0] += 1
        if "WARPGROUP.ARRIVE" in line:
            out[cur][1] += 1
        if "WARPGROUP.DEPBAR" in line:
            out[cur][2] += 1
    return out


def test_conv_tc_kernel_mmas_are_not_serialized(built_lib):
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    obj = os.path.join(os.path.dirname(built_lib), "conv_tc.o")
    sass = subprocess.run([tool, "-sass", obj], check=True, capture_output=True, text=True).stdout
    kernels = _kernels(sass)
    assert kernels, "no conv_tc_kernel instantiation in conv_tc.o"
    bad = []
    for (p1, p2, promo, ni, minb, tt), (hgmma, arrive, depbar) in sorted(kernels.items()):
        fused = p2 != -1
        # ARRIVE (static count): the wgmma.fence after the weight-slot wait, the head of the tap loop (its back edge:
        # once per tap, not per HGMMA), the commit, and the fused GEMM 2's batch -- 3 plain, 4 fused, however many
        # HGMMAs the class issues per tap.  A guarded batch gets one ARRIVE per HGMMA (up to 99 per instantiation).
        # DEPBAR: only the chunk-level wgmma.wait_group 0, one per GEMM.
        if hgmma == 0 or arrive > 4 or depbar > (2 if fused else 1):
            bad.append(f"conv_tc_kernel<{p1}, {p2}, {promo}, {ni}, {minb}, {tt}>: HGMMA {hgmma}, ARRIVE {arrive}, DEPBAR {depbar}")
    assert not bad, "wgmma serialized by ptxas:\n" + "\n".join(bad)
