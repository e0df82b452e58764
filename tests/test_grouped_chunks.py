"""The wgmma conv kernel steps through the K loop of a layer of 1-3 taps (1x1 convs, up- and down-sampling convs, the LSTM
input GEMMs) G = 2 or 4 sixteen-channel chunks at a time, so each step's barrier, weight wait, load round trip and
tensor-pipe drain is paid once per G chunks.  Every output element sums the same products in the same order as a
one-chunk step, with promotions at the same chunks, so the grouped launch equals the one-chunk launch bit for bit.

The host tests (no GPU) check the planner's G over every codec geometry; the GPU tests compare a grouped launch with the
same layer run one chunk per step (fac_debug_conv_tc_group1) and with fp64 torch.
"""
import ctypes
import math

import pytest
import torch

KEYS = ("N", "MT", "nchunk", "stages", "rows", "smem", "Rpad", "promote_every")
SMEM_CAP = 227 * 1024
SMEM_CAP2 = 113 * 1024


def _encoder():
    """(Cin, Cout, K, dil, stride, Tout) of config.yml's encoder convs at the bench length (test_host.py's list)."""
    enc, T, c = [], 96000, 64
    for s in (2, 5, 5, 6):
        for d in (1, 3, 9):
            enc += [(c, c, 7, d, 1, T), (c, c, 1, 1, 1, T)]
        enc.append((c, 2 * c, 2 * s, 1, s, T // s))
        T //= s
        c *= 2
    return enc + [(1024, 4096, 1, 1, 1, 320 * 32), (1024, 1024, 3, 1, 1, 320)]


def _decoder():
    """(Cin, Cout, K, dil, stride, Tout, mode) of the decoder's tensor-core layers at the bench length: 2 = bf16 split,
    7 = one fp16 pass (k = 7 convs), 8 = fused ResidualUnit."""
    dec, T, c = [], 320, 1536
    for s in (6, 5, 5, 2):
        dec.append((c, (c // 2) * s, 2, 1, 1, T, 2))                 # transposed conv as a 2-tap conv
        T *= s
        c //= 2
        for d in (1, 3, 9):
            if c <= 256:
                dec.append((c, c, 7, d, 1, T, 8))
            else:
                dec += [(c, c, 7, d, 1, T, 7), (c, c, 1, 1, 1, T, 2)]
    return dec + [(1024, 1536, 7, 1, 1, 320, 7), (1536, 6144, 1, 1, 1, 320 * 32, 2)]


def _plan(L, geom, mode):
    out = (ctypes.c_int * 8)()
    assert L.fac_debug_tc_plan(*geom, mode, 0, out) == 0, (geom, mode)
    g = L.fac_debug_tc_plan_group(*geom, mode, 0, None)
    assert g in (1, 2, 4), (geom, mode, g)
    return dict(zip(KEYS, list(out))), g


def test_group_divides_the_k_loop_and_keeps_the_residency(built_lib):
    """Every codec geometry: G divides the chunk count (and the promotion window of a promoted layer), and the grouped
    plan stays within the shared memory of its residency (half the SM for the promoted class)."""
    from facodec_b200 import _lib
    L = _lib.load()
    geoms = [(g, 3) for g in _encoder()] + [(g, 0) for g in _encoder() if g[2] == 1 and g[0] <= 128]
    geoms += [(tuple(d[:6]), d[6]) for d in _decoder()]
    for geom, mode in geoms:
        p, g = _plan(L, geom, mode)
        assert p["nchunk"] % g == 0, (geom, mode, p, g)
        if mode in (1, 3):
            assert p["promote_every"] % g == 0 and p["smem"] <= SMEM_CAP2, (geom, mode, p, g)
        assert p["smem"] <= SMEM_CAP, (geom, mode, p, g)


def test_grouping_never_costs_two_ctas_per_sm(built_lib):
    """A layer whose one-chunk plan fits half the shared memory (two CTAs per SM) keeps fitting it when grouped, in every
    class and with the "tc_occ2_maxn" option on or off; a grouped plan never exceeds the full 227 KB."""
    from facodec_b200 import _lib
    L = _lib.load()
    geoms = [(g, m) for g in _encoder() for m in (0, 1, 3) if g[2] <= 3 or g[4] > 1]
    geoms += [(tuple(d[:6]), m) for d in _decoder() if d[2] <= 3 for m in (0, 2)]
    geoms += [((c[2], c[3], c[4], c[5], c[6], _tout(c)), m) for c in CASES for m in (0, 1, 2, 3)]
    smem2 = (ctypes.c_int * 2)()
    grouped = 0
    for geom, mode in geoms:
        for occ2 in (0, 256):
            g = L.fac_debug_tc_plan_group(*geom, mode, occ2, smem2)
            assert g in (1, 2, 4), (geom, mode, occ2, g)
            grouped += g > 1
            if smem2[1] <= SMEM_CAP2:
                assert smem2[0] <= SMEM_CAP2, (geom, mode, occ2, g, list(smem2))
            assert smem2[0] <= SMEM_CAP, (geom, mode, occ2, g, list(smem2))
    assert grouped > 0


def test_short_tap_layers_are_grouped_and_k7_layers_are_not(built_lib):
    """k = 7 convs (and fused units, whose GEMM 1 is one) step one chunk at a time: their 7 taps of MMAs per chunk already
    cover the step's fixed cost.  The 1x1 convs, down-convs, up-convs and LSTM input GEMMs step 2-4 chunks, except the
    first decoder up-conv (C = 1536 at 320 frames), whose two-chunk weight slots would not fit two CTAs per SM."""
    from facodec_b200 import _lib
    L = _lib.load()
    for geom in _encoder():
        _, g = _plan(L, geom, 3)
        if geom[2] == 7:
            assert g == 1, geom
        elif geom[2] == 1 or geom[4] > 1:
            assert g > 1, geom
    for d in _decoder():
        geom, mode = tuple(d[:6]), d[6]
        _, g = _plan(L, geom, mode)
        if geom[2] == 7:
            assert g == 1, (geom, mode)
        elif geom[:2] != (1536, 4608):
            assert g > 1, (geom, mode)


def test_group1_debug_hook_rejects_missing_output(built_lib):
    from facodec_b200 import _lib
    L = _lib.load()
    assert L.fac_debug_conv_tc_group1(None, None, None, None, 1, 16, 16, 16, 1, 1, 1, 0, 0, 0, None, None, 0, None, None,
                                      16, 0, None, None) < 0


# ---- GPU --------------------------------------------------------------------------------------------------------------

CASES = [
    # B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, in_snake, out_snake, res
    (2, 150, 1024, 4096, 1, 1, 1, 0, 0, 0, 0, 0, 0),       # LSTM input GEMM, ragged Tout, two promotion windows (f16x2)
    (2, 100, 512, 1024, 12, 1, 6, 6, 5, 1, 1, 0, 0),       # stride-6 down-conv, Tout = 17
    (1, 203, 128, 256, 10, 1, 5, 5, 2, 1, 1, 0, 0),        # stride-5 down-conv, ragged
    (2, 333, 384, 384, 1, 1, 1, 0, 0, 0, 1, 1, 1),         # 1x1 with both Snakes and the residual
    (2, 700, 256, 256, 1, 1, 1, 0, 0, 1, 0, 0, 1),         # encoder 1x1 + residual
    (3, 20, 1536, 768, 2, 1, 1, 1, 0, 0, 1, 0, 0),         # transposed-conv form
    (1, 300, 384, 1920, 2, 1, 1, 1, 0, 0, 1, 0, 0),        # up-conv 384 -> 5 * 384
    (2, 70, 1024, 1024, 3, 1, 1, 2, 0, 1, 1, 0, 0),        # encoder conv_out, 3 taps: two-chunk slots exceed half the SM
    (2, 90, 1200, 2176, 1, 1, 1, 0, 0, 0, 0, 0, 0),        # Cin = 1200: 75 chunks, odd, so one chunk per step everywhere
    (3, 333, 64, 64, 1, 1, 1, 0, 0, 0, 1, 1, 1),           # encoder C = 64 1x1 (short chain: 3xTF32), ragged
    (2, 200, 64, 128, 4, 1, 2, 2, 0, 1, 1, 0, 0),          # stride-2 down-conv
]
# chunks per step the planner gives each case in the classes 0, 1, 2, 3 below: the GPU test runs exactly these
GROUPS = [(1, 1, 2, 2), (1, 1, 1, 2), (1, 1, 1, 2), (1, 1, 2, 4), (1, 1, 2, 4), (1, 1, 1, 2), (1, 1, 2, 2), (1, 1, 1, 1),
          (1, 1, 1, 1), (2, 2, 4, 4), (1, 1, 2, 2)]
# fac_debug_conv_tc classes: 0 = 3xTF32, 1 = promoted 3xTF32, 2 = bf16 split, 3 = promoted f16x2 (the one-pass fp16
# class runs the k = 7 convs, one chunk per step); fp64 tolerances (x scale) as test_gpu_kernels.py
TOL = {0: 6e-5, 1: 4e-6, 2: 2e-4, 3: 4e-6}


def _tout(case):
    T, K, dil, stride, pl, pr = case[1], case[4], case[5], case[6], case[7], case[8]
    return (T + pl + pr - ((K - 1) * dil + 1)) // stride + 1


def test_gpu_cases_plan_the_expected_groups(built_lib):
    """The GPU cases run grouped where GROUPS says so (no GPU needed to check the plans), with G > 1 in every class."""
    from facodec_b200 import _lib
    L = _lib.load()
    for c, want in zip(CASES, GROUPS):
        got = tuple(L.fac_debug_tc_plan_group(c[2], c[3], c[4], c[5], c[6], _tout(c), mode, 0, None) for mode in TOL)
        assert got == want, (c, got, want)
    for mode in TOL:
        assert max(want[mode] for want in GROUPS) > 1, mode


def _engine():
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    return e


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("case,groups", list(zip(CASES, GROUPS)))
def test_grouped_launch_equals_one_chunk_launch(case, groups, mode, built_lib):
    from test_gpu_kernels import ref_conv
    B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, ins, outs, res = case
    e = _engine()
    g = torch.Generator().manual_seed(hash(case) % 1000 + mode)
    x = torch.randn(B, Cin, T, generator=g) * 0.5
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    b = torch.randn(Cout, generator=g) * 0.1
    ia = (torch.rand(Cin, generator=g) + 0.5) if ins else None
    oa = (torch.rand(Cout, generator=g) + 0.5) if outs else None
    Tout = _tout(case)
    r = torch.randn(B, Cout, Tout, generator=g) if res else None
    xd = x.transpose(1, 2).contiguous().cuda()
    rd = r.transpose(1, 2).contiguous().cuda() if res else None
    args = (_p(xd), _p(w.contiguous()), _p(b), B, T, Cin, Cout, K, dil, stride, pl, pr, reflect, _p(ia), _p(oa), 0, _p(rd))
    y1 = torch.full((B, Tout, Cout), float("nan"), device="cuda")
    yg = torch.full((B, Tout, Cout), float("nan"), device="cuda")
    group = ctypes.c_int(0)
    rc = e.L.fac_debug_conv_tc_group1(e.handle, *args, _p(y1), Tout, mode, None, ctypes.byref(group))
    assert rc == 0, e.L.fac_last_error(e.handle)
    rc = e.L.fac_debug_conv_tc(e.handle, *args, _p(yg), Tout, mode, None)
    assert rc == 0, e.L.fac_last_error(e.handle)
    y1, yg = y1.cpu(), yg.cpu()
    assert group.value == groups[mode], (case, mode, group.value)
    assert torch.equal(yg, y1), f"G = {group.value}: grouped launch differs from the one-chunk launch"
    ref = ref_conv(x, w, b, dil, stride, pl, pr, reflect, ia, oa, 0, r)
    y = yg.transpose(1, 2).double()
    assert torch.isfinite(y).all()
    err = (y - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"GROUP mode={mode} G={group.value} case={case} maxerr={err:.3e} scale={scale:.3f}")
    assert err <= TOL[mode] * max(scale, 1.0), f"max err {err} (scale {scale})"
