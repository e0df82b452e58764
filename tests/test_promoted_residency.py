"""The promoted wgmma conv class (layers upstream of the VQ) runs two CTAs per SM.

Its fp32 master accumulator lives in shared memory, so a thread holds only the current window's accumulators: <= 128
registers.  The host tests (no GPU) check the tile plans and the compiled kernels' resources; the GPU tests check the
multi-window promotion through shared memory against an fp64 reference.
"""
import ctypes
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

KEYS = ("N", "MT", "nchunk", "stages", "rows", "smem", "Rpad", "promote_every")
SMEM_CAP2 = 113 * 1024          # dynamic shared memory per block with two resident blocks per SM (sm_90)


def _encoder_geometries():
    """(Cin, Cout, K, dil, stride, Tout) of every promoted conv of config.yml's encoder at the bench length, the LSTM
    input GEMM and the final k = 3 conv (as in test_host.py::test_tile_plans_of_every_codec_layer_fit_the_sm)."""
    enc = []
    T, c = 96000, 64
    for s in (2, 5, 5, 6):
        for d in (1, 3, 9):
            enc += [(c, c, 7, d, 1, T), (c, c, 1, 1, 1, T)]
        enc.append((c, 2 * c, 2 * s, 1, s, T // s))
        T //= s
        c *= 2
    return enc + [(1024, 4096, 1, 1, 1, 320 * 32), (1024, 1024, 3, 1, 1, 320)]


def _plan(L, geom, mode):
    out = (ctypes.c_int * 8)()
    assert L.fac_debug_tc_plan(*geom, mode, 0, out) == 0, (geom, mode)
    return dict(zip(KEYS, list(out)))


def test_promoted_encoder_layers_plan_two_ctas_per_sm(built_lib):
    """fp16 hi + scaled-lo class (mode 3, the default upstream of the VQ): every encoder geometry fits two CTAs per SM, with
    the tile width N the weight blob was laid out for (64 at C = 64, else 128)."""
    from facodec_b200 import _lib
    L = _lib.load()
    for g in _encoder_geometries():
        p = _plan(L, g, 3)
        assert p["N"] == (64 if g[1] == 64 else 128), g
        assert p["smem"] <= SMEM_CAP2, (g, p)


def test_tf32_promoted_layers_fall_back_to_one_cta_only_when_they_must(built_lib):
    """3xTF32 class (mode 1): its weight slot is twice the fp16 one, so the k = 7 convs at N = 128 cannot fit two CTAs (one
    slot alone is 112 KB); every other geometry must.  N is unchanged by the residency."""
    from facodec_b200 import _lib
    L = _lib.load()
    for g in _encoder_geometries():
        p = _plan(L, g, 1)
        assert p["N"] == (64 if g[1] == 64 else 128), g
        if g[2] == 7 and p["N"] == 128:
            assert p["smem"] > SMEM_CAP2, (g, p)
        else:
            assert p["smem"] <= SMEM_CAP2, (g, p)


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if c and os.path.exists(c):
            return c
    return None


def test_promoted_kernels_fit_two_ctas_without_spills(built_lib):
    """Every promoted instantiation but the transposed one is compiled for two CTAs per SM (MINB = 2) and fits it: <= 128
    registers and no local memory.  The stack frame stays at the 32 bytes the fp32-operand instantiations all have (an
    addressable array, no spill); a register spill would grow it."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    obj = os.path.join(os.path.dirname(built_lib), "conv_tc.o")
    out = subprocess.run([tool, "-res-usage", obj], check=True, capture_output=True, text=True).stdout
    kernels, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            t = re.search(r"conv_tc_kernelI((?:L[ib]n?\d+E)+)E", m.group(1))
            cur = tuple(int(v) * (-1 if n else 1) for _, n, v in re.findall(r"L([ib])(n?)(\d+)E", t.group(1))) if t else None
            continue
        if cur is not None and "REG:" in line:
            kernels[cur] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", line)}
            cur = None
    promoted = {k: v for k, v in kernels.items() if k[2] == 1 and not k[5]}       # (P1, P2, PROMO, NI, MINB, TT)
    assert {(k[0], k[3]) for k in promoted} == {(p1, ni) for p1 in (0, 3) for ni in (16, 32, 48, 64)}
    for k, r in sorted(promoted.items()):
        assert k[4] == 2, f"conv_tc_kernel{k}: promoted class compiled for one CTA per SM"
        assert r["REG"] <= 128 and r["LOCAL"] == 0 and r["STACK"] <= 32, f"conv_tc_kernel{k}: {r}"


# ---- GPU --------------------------------------------------------------------------------------------------------------

CASES = [
    # B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, in_snake, out_snake, res      windows (f16x2 / tf32)
    (2, 260, 512, 512, 7, 9, 1, 54, 0, 1, 1, 1, 0),      # 6 / 32, ragged Tout
    (2, 150, 1024, 4096, 1, 1, 1, 0, 0, 0, 0, 0, 0),     # 2 / 8, LSTM input GEMM geometry
    (2, 100, 512, 1024, 12, 1, 6, 6, 5, 1, 1, 0, 0),     # 8 / 48, stride-6 down-conv, Tout = 17
    (3, 333, 64, 64, 7, 3, 1, 18, 0, 1, 1, 1, 1),        # 1 / 4, C = 64 k7 + residual: no master in the f16x2 class
    (2, 70, 1024, 1024, 3, 1, 1, 2, 0, 1, 1, 0, 0),      # 4 / 32, encoder conv_out
]


def _engine():
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    return e


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _run(e, case, mode, seed):
    B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, ins, outs, res = case
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, T, generator=g) * 0.5
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g) * 0.1
    ia = (torch.rand(Cin, generator=g) + 0.5) if ins else None
    oa = (torch.rand(Cout, generator=g) + 0.5) if outs else None
    Tout = (T + pl + pr - ((K - 1) * dil + 1)) // stride + 1
    r = torch.randn(B, Cout, Tout, generator=g) if res else None
    xd = x.transpose(1, 2).contiguous().cuda()
    rd = r.transpose(1, 2).contiguous().cuda() if res else None
    outs_ = []
    for _ in range(2):
        yd = torch.full((B, Tout, Cout), float("nan"), device="cuda")
        rc = e.L.fac_debug_conv_tc(e.handle, _p(xd), _p(w.contiguous()), _p(b), B, T, Cin, Cout, K, dil, stride, pl, pr,
                                   reflect, _p(ia), _p(oa), 0, _p(rd), _p(yd), Tout, mode, None)
        assert rc == 0, e.L.fac_last_error(e.handle)
        outs_.append(yd.cpu())
    return (x, w, b, dil, stride, pl, pr, reflect, ia, oa, 0, r), outs_


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [3, 1, 4])
@pytest.mark.parametrize("case", CASES)
def test_promoted_conv_vs_fp64(case, mode, built_lib):
    """Promotion windows summed in the shared-memory master, against fp64 torch, at the 4e-6 x scale bound the promoted
    class is held to (test_gpu_kernels.py::test_conv_tc_kernel_vs_torch); 3 = fp16 hi + scaled lo (two CTAs per SM),
    1 = 3xTF32, 4 = the transposed formulation of 3.  Two calls give the same bits."""
    from test_gpu_kernels import ref_conv
    e = _engine()
    args, (y0, y1) = _run(e, case, mode, hash(case) % 1000 + mode)
    assert torch.equal(y0, y1), "repeated calls differ"
    ref = ref_conv(*args)
    y = y0.transpose(1, 2).double()
    assert torch.isfinite(y).all()
    err = (y - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"PROMO mode={mode} case={case} maxerr={err:.3e} scale={scale:.3f}")
    assert err <= 4e-6 * max(scale, 1.0), f"max err {err} (scale {scale})"
