"""The one-pass fp16 conv class (the decoder's k = 7 convs) runs the tiles whose 64-row plan would hold one CTA per SM as
128 rows, each warpgroup over all N channels (wgmma m64n256 plain, m64n192 fused), so both warpgroups share every weight
chunk streamed into shared memory.

The host tests (no GPU) pin the plans of the decoder's ResidualUnits and the compiled kernels' resources; the GPU tests
check the wide tiles against an fp64 reference.
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
SMEM_CAP = 227 * 1024           # dynamic shared memory per block on sm_90
SMEM_CAP2 = 113 * 1024          # ... with two resident blocks per SM
PLAIN, FUSED = 7, 8             # fac_debug_tc_plan modes of the one-pass fp16 class


def _plan(L, geom, mode, occ2=0):
    out = (ctypes.c_int * 8)()
    assert L.fac_debug_tc_plan(*geom, mode, occ2, out) == 0, (geom, mode)
    return dict(zip(KEYS, list(out)))


def _nw(p):
    return p["N"] if p["MT"] == 2 else p["N"] // 2


def test_decoder_residual_units_plan_128_row_tiles(built_lib):
    """At the bench lengths: the C = 768 conv7 (plain) and the C = 192 unit (fused) take 128-row tiles at the N the weight
    blobs were laid out for; the C = 384 conv7 keeps its 64-row tiles (two CTAs per SM) and the C = 96 unit its 128 rows of
    N = 96.  The bf16 classes' N (the 1x1 convs, and the unfused plan a fused unit's blobs come from) is the same N."""
    from facodec_b200 import _lib
    L = _lib.load()
    want = {(768, PLAIN): (256, 2), (384, PLAIN): (192, 1), (192, FUSED): (192, 2), (96, FUSED): (96, 2)}
    T = {768: 1920, 384: 9600, 192: 48000, 96: 96000}
    for (C, mode), (N, MT) in want.items():
        for d in (1, 3, 9):
            g = (C, C, 7, d, 1, T[C])
            p = _plan(L, g, mode)
            assert (p["N"], p["MT"], p["rows"], p["nchunk"]) == (N, MT, 64 * MT, C // 16), (g, p)
            assert _nw(p) <= 256 and p["smem"] <= SMEM_CAP and p["stages"] == 2, (g, p)
            if MT == 1:
                assert p["smem"] <= SMEM_CAP2, (g, p)
            assert _plan(L, g, 2)["N"] == N and _plan(L, (C, C, 1, 1, 1, T[C]), 2)["N"] == N
            assert _plan(L, g, 7)["N"] == N


def test_wide_tiles_only_at_compiled_widths(built_lib):
    """Over every 16-channel width up to 1024, the one-pass class's warpgroup width is <= 128 or the width its kernel is
    compiled for (256 plain, 192 fused), the latter only where the 64-row plan would not fit two CTAs per SM; a plan for
    two CTAs per SM ("tc_occ2_maxn") is never wide."""
    from facodec_b200 import _lib
    L = _lib.load()
    for C in range(16, 1025, 16):
        p = _plan(L, (C, C, 7, 3, 1, 4096), PLAIN)
        assert _nw(p) <= 128 or (_nw(p) == 256 and p["rows"] == 128), (C, p)
        assert p["rows"] == 64 * p["MT"] and p["smem"] <= SMEM_CAP
        if C <= 256:
            q = _plan(L, (C, C, 7, 3, 1, 4096), FUSED)
            assert _nw(q) <= 128 or _nw(q) == 192, (C, q)
            assert q["smem"] <= SMEM_CAP
        p2 = _plan(L, (C, C, 7, 3, 1, 4096), PLAIN, occ2=256)
        assert _nw(p2) <= 64 or p2 == p, (C, p2)        # two CTAs per SM, or the one-CTA plan


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if c and os.path.exists(c):
            return c
    return None


def test_wide_one_pass_kernels_do_not_spill(built_lib):
    """Every one-pass fp16 instantiation wider than 128 columns (an m64n256 / fused m64n192 accumulator: 128 / 96 registers
    per thread) is compiled for one CTA per SM and fits it without local memory."""
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
    wide = {k: v for k, v in kernels.items() if k[0] == 2 and k[3] > 128}      # (P1, P2, PROMO, NI, MINB, TT), P_F16S = 2
    assert {(k[1], k[3]) for k in wide} == {(-1, 256), (1, 192)}
    for k, r in sorted(wide.items()):
        assert k[4] == 1, f"conv_tc_kernel{k}: wide tile compiled for two CTAs per SM"
        assert r["LOCAL"] == 0 and r["REG"] <= 255, f"conv_tc_kernel{k}: {r}"


# ---- GPU --------------------------------------------------------------------------------------------------------------

CONV_CASES = [
    # B, T, C, dil, pl, res                128-row tiles
    (2, 300, 256, 1, 6, 0),             # 3 tiles with a ragged tail
    (3, 700, 768, 3, 18, 1),            # 3 channel tiles x 6 time tiles, residual
    (2, 40, 256, 9, 54, 0),             # input shorter than the receptive field (reflect branch)
    (1, 1000, 512, 9, 54, 1),           # 2 channel tiles x 8 time tiles, residual
]


def _engine():
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    return e


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONV_CASES)
def test_wide_one_pass_conv_vs_fp64(case, built_lib):
    """k = 7 conv with both Snakes through the one-pass fp16 class (fac_debug_conv_tc mode 5) on a wide tile, against fp64
    torch at that class's tolerance (test_gpu_kernels.py::test_conv_tc_kernel_vs_torch); two calls give the same bits."""
    from test_gpu_kernels import ref_conv
    B, T, C, dil, pl, res = case
    e = _engine()
    e.set_option("tc_occ2_maxn", 0)
    p = _plan(e.L, (C, C, 7, dil, 1, T), PLAIN)
    assert p["MT"] == 2 and p["N"] > 128, p
    g = torch.Generator().manual_seed(C + dil + T)
    x = torch.randn(B, C, T, generator=g) * 0.5
    w = torch.randn(C, C, 7, generator=g) / math.sqrt(C * 7)
    b = torch.randn(C, generator=g) * 0.1
    ia = torch.rand(C, generator=g) + 0.5
    oa = torch.rand(C, generator=g) + 0.5
    r = torch.randn(B, C, T, generator=g) if res else None
    xd = x.transpose(1, 2).contiguous().cuda()
    rd = r.transpose(1, 2).contiguous().cuda() if res else None
    ys = []
    for _ in range(2):
        yd = torch.full((B, T, C), float("nan"), device="cuda")
        rc = e.L.fac_debug_conv_tc(e.handle, _p(xd), _p(w.contiguous()), _p(b), B, T, C, C, 7, dil, 1, pl, 0, 1,
                                   _p(ia), _p(oa), 0, _p(rd), _p(yd), T, 5, None)
        assert rc == 0, e.L.fac_last_error(e.handle)
        ys.append(yd.cpu())
    assert torch.equal(ys[0], ys[1]), "repeated calls differ"
    ref = ref_conv(x, w, b, dil, 1, pl, 0, 1, ia, oa, 0, r)
    y = ys[0].transpose(1, 2).double()
    assert torch.isfinite(y).all()
    err = (y - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"WIDE conv case={case} maxerr={err:.3e} scale={scale:.3f}")
    assert err <= 2e-3 * max(scale, 1.0), f"max err {err} (scale {scale})"


UNIT_CASES = [
    # B, T, C, dil, mode (6: fused unit, 5: conv7 + conv1 launches)
    (2, 300, 192, 9, 6),                # fused C = 192, ragged tail
    (3, 1000, 192, 1, 6),
    (2, 40, 192, 9, 6),                 # input shorter than the receptive field
    (2, 300, 768, 3, 5),                # conv7 on N = 256 wide tiles, then the bf16 1x1
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", UNIT_CASES)
def test_wide_residual_unit_vs_fp64(case, built_lib):
    """Whole ResidualUnit (fac_debug_resunit) with its k = 7 conv on a wide one-pass tile, against the fp64 oracle at the
    tolerance of test_gpu_kernels.py::test_residual_unit_modes modes 5 / 6; two calls give the same bits."""
    from oracle import facodec_oracle as O
    B, T, C, dil, mode = case
    e = _engine()
    e.set_option("tc_occ2_maxn", 0)
    p = _plan(e.L, (C, C, 7, dil, 1, T), FUSED if mode == 6 else PLAIN)
    assert p["MT"] == 2 and p["N"] > 128, p
    g = torch.Generator().manual_seed(C + dil + T + mode)
    x = torch.randn(B, C, T, generator=g) * 0.5
    w7 = torch.randn(C, C, 7, generator=g) / math.sqrt(C * 7)
    w1 = torch.randn(C, C, 1, generator=g) / math.sqrt(C)
    b7 = torch.randn(C, generator=g) * 0.1
    b1 = torch.randn(C, generator=g) * 0.1
    a1 = torch.rand(C, generator=g) + 0.5
    a2 = torch.rand(C, generator=g) + 0.5
    sd = {"u.block.0.alpha": a1.view(1, C, 1), "u.block.1.conv.conv.weight": w7, "u.block.1.conv.conv.bias": b7,
          "u.block.2.alpha": a2.view(1, C, 1), "u.block.3.conv.conv.weight": w1, "u.block.3.conv.conv.bias": b1}
    ref = O.residual_unit(x.double(), {k: v.double() for k, v in sd.items()}, "u", dil)
    xd = x.transpose(1, 2).contiguous().cuda()
    ys = []
    for _ in range(2):
        yd = torch.full((B, T, C), float("nan"), device="cuda")
        rc = e.L.fac_debug_resunit(e.handle, _p(xd), _p(w7.contiguous()), _p(b7), _p(w1.contiguous()), _p(b1), _p(a1),
                                   _p(a2), B, T, C, dil, mode, _p(yd), None)
        assert rc == 0, e.L.fac_last_error(e.handle)
        ys.append(yd.cpu())
    assert torch.equal(ys[0], ys[1]), "repeated calls differ"
    y = ys[0].transpose(1, 2).double()
    assert torch.isfinite(y).all()
    err = (y - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"WIDE unit case={case} maxerr={err:.3e} scale={scale:.3f}")
    assert err <= 2e-3 * max(scale, 1.0), f"max err {err} (scale {scale})"
