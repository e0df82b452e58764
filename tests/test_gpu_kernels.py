"""GPU: kernel-level parity through the C-ABI test hooks (fac_debug_conv / fac_debug_conv_tc / fac_debug_resunit_lanes)
against plain PyTorch on CPU -- the same functional calls the oracle restatement uses.  The LSTM recurrence has its own
fp64 suite in test_gpu_lstm.py."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _engine():
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    return e


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def ref_conv(x, w, b, dil, stride, pl, pr, reflect, in_alpha, out_alpha, act, res):
    """x [B,Cin,T] (NCT) torch reference with the oracle's padding helper, in float64: the promoted kernels are held to
    4e-6 of scale, about the error of an fp32 CPU conv over K*Cin = 7168 terms, so the reference must not add its own."""
    from oracle import facodec_oracle as O
    x, w = x.double(), w.double()
    b = b.double() if b is not None else None
    in_alpha = in_alpha.double() if in_alpha is not None else None
    out_alpha = out_alpha.double() if out_alpha is not None else None
    res = res.double() if res is not None else None
    if in_alpha is not None:
        x = O.snake(x, in_alpha.view(1, -1, 1))
    if reflect:
        x = O._pad1d_reflect(x, pl, pr)
    else:
        x = F.pad(x, (pl, pr))
    y = F.conv1d(x, w, b, stride=stride, dilation=dil)
    if out_alpha is not None:
        y = O.snake(y, out_alpha.view(1, -1, 1))
    if act == 1:
        y = torch.tanh(y)
    elif act == 2:
        y = y * torch.tanh(F.softplus(y))
    if res is not None:
        y = y + res
    return y


CASES = [
    # B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, in_snake, out_snake, act, res
    (2, 300, 1, 64, 7, 1, 1, 6, 0, 1, 0, 0, 0, 0),        # encoder conv0 (conv_cin1_kernel)
    (1, 1031, 1, 64, 7, 1, 1, 6, 0, 1, 0, 0, 0, 0),       # ... several CTAs, ragged tail
    (2, 5, 1, 64, 7, 1, 1, 6, 0, 1, 0, 0, 0, 0),          # ... short-input reflect branch (L <= pad)
    (1, 600, 1, 32, 3, 2, 1, 4, 0, 0, 0, 0, 1, 0),        # ... dilated, zero pad, tanh, 32 channels
    (2, 4000, 96, 1, 7, 1, 1, 6, 0, 1, 1, 0, 1, 0),       # final conv + tanh over several CTAs (conv_cout1_kernel)
    (2, 333, 64, 64, 7, 1, 1, 6, 0, 1, 1, 1, 0, 0),       # residual conv7 d=1
    (1, 200, 64, 64, 7, 9, 1, 54, 0, 1, 1, 1, 0, 0),      # d=9
    (2, 40, 96, 96, 7, 9, 1, 54, 0, 1, 1, 1, 0, 0),       # short-input reflect branch (L <= pad), BN=96
    (2, 150, 128, 128, 1, 1, 1, 0, 0, 1, 0, 0, 0, 1),     # residual conv1 + skip
    (2, 200, 64, 128, 4, 1, 2, 2, 0, 1, 1, 0, 0, 0),      # down conv s=2
    (1, 203, 128, 256, 10, 1, 5, 5, 2, 1, 1, 0, 0, 0),    # down conv s=5 with extra right pad (ragged)
    (1, 37, 512, 1024, 12, 1, 6, 6, 5, 1, 1, 0, 0, 0),    # s=6 ragged
    (2, 50, 192, 192, 7, 3, 1, 18, 0, 1, 1, 1, 0, 0),     # BN=96 x2
    (2, 64, 96, 1, 7, 1, 1, 6, 0, 1, 1, 0, 1, 0),         # final conv + tanh, Cout=1
    (2, 31, 80, 512, 1, 1, 1, 0, 0, 0, 0, 0, 2, 0),       # StyleEncoder 1x1 + Mish
    (2, 31, 512, 1024, 5, 1, 1, 2, 2, 0, 0, 0, 0, 0),     # Conv1dGLU conv (zero pad both sides)
    (1, 9000, 1, 2050, 1200, 1, 300, 600, 600, 1, 0, 0, 0, 0),  # STFT-as-conv geometry
    (3, 20, 1536, 768, 2, 1, 1, 1, 0, 0, 1, 0, 0, 0),     # transposed-conv form (zero left pad)
]


@pytest.mark.parametrize("case", CASES)
def test_conv_kernel_vs_torch(case, built_lib):
    B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, ins, outs, act, res = case
    e = _engine()
    g = torch.Generator().manual_seed(hash(case) % 1000)
    x = torch.randn(B, Cin, T, generator=g) * 0.5
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g) * 0.1
    ia = (torch.rand(Cin, generator=g) + 0.5) if ins else None
    oa = (torch.rand(Cout, generator=g) + 0.5) if outs else None
    Tout = (T + pl + pr - ((K - 1) * dil + 1)) // stride + 1
    r = torch.randn(B, Cout, Tout, generator=g) if res else None
    ref = ref_conv(x, w, b, dil, stride, pl, pr, reflect, ia, oa, act, r)
    assert ref.shape[-1] == Tout
    xd = x.transpose(1, 2).contiguous().cuda()
    rd = r.transpose(1, 2).contiguous().cuda() if res else None
    yd = torch.empty(B, Tout, Cout, device="cuda")
    rc = e.L.fac_debug_conv(e.handle, _p(xd), _p(w.contiguous()), _p(b), B, T, Cin, Cout, K, dil, stride, pl, pr, reflect,
                            _p(ia), _p(oa), act, _p(rd), _p(yd), Tout, None)
    assert rc == 0, e.L.fac_last_error(e.handle)
    y = yd.cpu().transpose(1, 2)
    err = (y - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 2e-5 * max(scale, 1.0), f"max err {err} (scale {scale})"


TC_CASES = [
    # B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, in_snake, out_snake, act, res
    (1, 128, 16, 64, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),       # one chunk, one tap, one N tile
    (1, 512, 64, 64, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),       # MT=4 full, 4 chunks
    (2, 300, 64, 64, 7, 1, 1, 6, 0, 1, 0, 0, 0, 0),       # taps as descriptor row offsets
    (2, 333, 64, 64, 7, 1, 1, 6, 0, 1, 1, 1, 0, 0),       # + snake prologue/epilogue
    (1, 700, 64, 64, 7, 9, 1, 54, 0, 1, 1, 1, 0, 0),      # d=9
    (2, 40, 96, 96, 7, 9, 1, 54, 0, 1, 1, 1, 0, 0),       # short-input reflect branch, N=96
    (2, 150, 128, 128, 1, 1, 1, 0, 0, 1, 0, 0, 0, 1),     # residual add
    (2, 200, 64, 128, 4, 1, 2, 2, 0, 1, 1, 0, 0, 0),      # down conv s=2 (vf=2)
    (1, 203, 128, 256, 10, 1, 5, 5, 2, 1, 1, 0, 0, 0),    # down conv s=5 ragged, N=256 MT=2
    (1, 37, 512, 1024, 12, 1, 6, 6, 5, 1, 1, 0, 0, 0),    # s=6 ragged, 4 N tiles
    (2, 260, 192, 192, 7, 3, 1, 18, 0, 1, 1, 1, 0, 0),    # N=192
    (2, 31, 512, 1024, 5, 1, 1, 2, 2, 0, 0, 0, 0, 0),     # zero pad both sides
    (3, 20, 1536, 768, 2, 1, 1, 1, 0, 0, 1, 0, 0, 0),     # transposed-conv form, N=256 x3
    (1, 300, 384, 1920, 2, 1, 1, 1, 0, 0, 1, 0, 0, 0),    # up-conv 384 -> 5*384, N=240
    (2, 64, 1024, 1024, 3, 1, 1, 2, 0, 1, 1, 0, 0, 0),    # encoder conv_out geometry
    (1, 640, 1024, 4096, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),   # LSTM input projection geometry
    (2, 320, 256, 512, 5, 1, 1, 4, 0, 1, 0, 0, 0, 0),     # WN in_layer geometry, T' = 320
    (1, 1000, 128, 128, 7, 3, 1, 18, 0, 1, 1, 1, 0, 1),   # several time tiles + residual + both Snakes
    (2, 700, 256, 256, 1, 1, 1, 0, 0, 1, 0, 0, 0, 1),     # encoder 1x1 + residual, two channel tiles, ragged tail
    (1, 1000, 64, 512, 3, 1, 1, 2, 0, 1, 1, 1, 0, 0),     # 3 taps, 4 channel tiles (two pairs), both Snakes, several time tiles
    (2, 300, 768, 768, 7, 1, 1, 6, 0, 1, 1, 1, 0, 0),     # decoder conv7 at C = 768: single-slot weight ring (stages == 1)
]


@pytest.mark.parametrize("occ2", [0, 256])
@pytest.mark.parametrize("promoted", [0, 1, 2, 3, 4, 5])
@pytest.mark.parametrize("case", TC_CASES)
def test_conv_tc_kernel_vs_torch(case, promoted, occ2, built_lib):
    """wgmma 3xTF32 conv vs fp32 torch.  Operands are split exactly (hi + lo), but the tensor core adds into its fp32
    accumulator with truncation, so the error grows with the number of chained MMAs; tolerance 6e-5 * scale.
    promoted=1 adds each window of <= 48 chained MMAs into an fp32 master accumulator: held to 4e-6 * scale like the
    fp32 FMA kernel."""
    B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, ins, outs, act, res = case
    if occ2 and promoted in (1, 3, 4):
        pytest.skip("the promoted kernel has a single residency plan")
    e = _engine()
    e.set_option("tc_occ2_maxn", occ2)      # 256: tiles planned for two resident CTAs per SM
    g = torch.Generator().manual_seed(hash(case) % 1000 + 7)
    x = torch.randn(B, Cin, T, generator=g) * 0.5
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g) * 0.1
    ia = (torch.rand(Cin, generator=g) + 0.5) if ins else None
    oa = (torch.rand(Cout, generator=g) + 0.5) if outs else None
    Tout = (T + pl + pr - ((K - 1) * dil + 1)) // stride + 1
    r = torch.randn(B, Cout, Tout, generator=g) if res else None
    ref = ref_conv(x, w, b, dil, stride, pl, pr, reflect, ia, oa, act, r)
    xd = x.transpose(1, 2).contiguous().cuda()
    rd = r.transpose(1, 2).contiguous().cuda() if res else None
    yd = torch.full((B, Tout, Cout), float("nan"), device="cuda")
    rc = e.L.fac_debug_conv_tc(e.handle, _p(xd), _p(w.contiguous()), _p(b), B, T, Cin, Cout, K, dil, stride, pl, pr, reflect,
                               _p(ia), _p(oa), act, _p(rd), _p(yd), Tout, promoted, None)
    assert rc == 0, e.L.fac_last_error(e.handle)
    y = yd.cpu().transpose(1, 2)
    assert torch.isfinite(y).all()
    err = (y - ref).abs().max().item()
    scale = ref.abs().max().item()
    rel_rms = ((y - ref).double().pow(2).mean().sqrt() / ref.double().pow(2).mean().sqrt()).item()
    print(f"TCERR promoted={promoted} occ2={occ2} case={case} maxerr={err:.3e} scale={scale:.3f} rel_rms={rel_rms:.3e}")
    # 3xTF32 / promoted (fp32-grade) / bf16 hi+lo / promoted with the fp16 hi + scaled-lo split (fp32-grade)
    # 4 = the transposed formulation of 3: weights as the wgmma A operand, time as wgmma N
    # 5 = ONE fp16 pass (the k = 7 convs downstream of the VQ): 10-bit operands, error ~2e-4 of the output's RMS
    tol = {0: 6e-5, 1: 4e-6, 2: 2e-4, 3: 4e-6, 4: 4e-6, 5: 2e-3}[promoted]
    assert err <= tol * max(scale, 1.0), f"max err {err} (scale {scale})"


UNIT_SHAPES = [(2, 300, 96, 1), (1, 520, 96, 9), (2, 200, 192, 3), (1, 130, 256, 1), (2, 40, 96, 9),
               (1, 700, 64, 3), (2, 300, 192, 9),     # C = 192, d = 9: single-slot ring
               (2, 20, 96, 9)]                        # T <= 27: the short-input branch of the non-causal split too


@pytest.mark.parametrize("occ2", [0, 256])
@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4, 5, 6])
@pytest.mark.parametrize("B,T,C,dil,causal", [pytest.param(*s, cz, id="-".join(map(str, s)) + ("" if cz else "-noncausal"))
                                              for s in UNIT_SHAPES for cz in (True, False)])
def test_residual_unit_modes(B, T, C, dil, causal, mode, occ2, built_lib):
    """ResidualUnit (dac.py:25-42) through the fp32 FMA path (0), two tensor-core launches (1 tf32, 3 bf16 split), and the
    fused launch (2 tf32, 4 bf16 split), 5/6 = 3/4 with the k = 7 conv in ONE fp16 pass (the product's default downstream of
    the VQ); occ2 = tiles planned for two CTAs per SM.  causal = False: the redecoder's decoder, reflected at both ends
    (pad (k_eff - 1) - (k_eff - 1) // 2 on the left, the rest on the right)."""
    from oracle import facodec_oracle as O
    if occ2 and mode == 0:
        pytest.skip("fp32 FMA path has no residency option")
    e = _engine()
    e.set_option("tc_occ2_maxn", occ2)
    g = torch.Generator().manual_seed(C + dil + T)
    x = torch.randn(B, C, T, generator=g) * 0.5
    w7 = torch.randn(C, C, 7, generator=g) / math.sqrt(C * 7)
    w1 = torch.randn(C, C, 1, generator=g) / math.sqrt(C)
    b7 = torch.randn(C, generator=g) * 0.1
    b1 = torch.randn(C, generator=g) * 0.1
    a1 = torch.rand(C, generator=g) + 0.5
    a2 = torch.rand(C, generator=g) + 0.5
    sd = {"u.block.0.alpha": a1.view(1, C, 1), "u.block.1.conv.conv.weight": w7, "u.block.1.conv.conv.bias": b7,
          "u.block.2.alpha": a2.view(1, C, 1), "u.block.3.conv.conv.weight": w1, "u.block.3.conv.conv.bias": b1}
    ref = O.residual_unit(x.double(), {k: v.double() for k, v in sd.items()}, "u", dil, causal=causal)
    xd = x.transpose(1, 2).contiguous().cuda()
    yd = torch.full((B, T, C), float("nan"), device="cuda")
    rc = e.L.fac_debug_resunit_lanes(e.handle, _p(xd), _p(w7.contiguous()), _p(b7), _p(w1.contiguous()), _p(b1), _p(a1),
                                     _p(a2), B, T, C, dil, mode, int(causal), None, _p(yd), None)
    if mode == 2 and C > 128:
        # the fused kernel keeps the whole GEMM-2 operand and a chunk's weights in shared memory: with the tf32 split
        # that only fits up to C = 128 (the product runs fused units with the bf16 split, mode 4)
        assert rc != 0
        return
    assert rc == 0, e.L.fac_last_error(e.handle)
    y = yd.cpu().transpose(1, 2)
    assert torch.isfinite(y).all()
    err = (y.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    tol = 2e-5 if mode == 0 else (8e-5 if mode <= 2 else (3e-4 if mode <= 4 else 2e-3))
    print(f"RESUNIT mode={mode} C={C} d={dil} T={T} causal={causal} maxerr={err:.3e} scale={scale:.3f}")
    assert err <= tol * max(scale, 1.0), f"max err {err} (scale {scale})"
