"""Builds the in-tree C-ABI shared library with nvcc for sm_90a.

    python -m facodec_b200.build            # build if stale
    python -m facodec_b200.build --force

Output: facodec_b200/_C/libfacodec_b200.so (git-ignored, rebuilt when a source is newer).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_C")
LIB = os.path.join(OUT_DIR, "libfacodec_b200.so")
SOURCES = ["engine.cu", "conv_simt.cu", "conv_tc.cu", "lstm.cu", "lstm2.cu", "frontend.cu", "quant.cu", "altfree.cu", "pool.cu", "resample.cu", "jdc.cu"]
HEADERS = ["common.cuh", "kernels.h", "conv_tc_common.cuh", "resample.h", os.path.join("..", "..", "include", "facodec_b200.h"),
           os.path.join("..", "..", "include", "facodec_b200_debug.h")]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-O3", "--expt-relaxed-constexpr"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    if not force and not is_stale():
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    objs = []
    procs = []
    for s in SOURCES:
        obj = os.path.join(OUT_DIR, s.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, s), "-o", obj]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    fail = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- {s} ---\n{out}\n")
        fail |= p.returncode != 0
    if fail:
        raise RuntimeError("nvcc failed")
    cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
