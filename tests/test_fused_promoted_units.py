"""The encoder's 64- and 128-channel ResidualUnits run as one fused launch in the promoted fp16 hi + scaled-lo class.

The fused launch keeps the k = 7 conv's Snake'd output on chip instead of writing it to global memory and reading it
back in a second launch.  It runs the same K loop, MMA shapes and promotion windows as the two launches, and splits the
same fp32 values for the 1x1, so its output is theirs bit for bit.  The host tests (no GPU) check the plans; the GPU
tests check that bit-equality for single units and through Codec.encode.
"""
import ctypes
import math

import pytest
import torch

KEYS = ("N", "MT", "nchunk", "stages", "rows", "smem", "Rpad", "promote_every")
SMEM_CAP2 = 113 * 1024          # dynamic shared memory per block with two resident blocks per SM (sm_90)
FAC_ERR_UNSUPPORTED = -4
PLAIN, FUSED_UNIT = 3, 9        # fac_debug_tc_plan modes: promoted fp16 hi + scaled lo, and its fused ResidualUnit
TWO_LAUNCHES, ONE_LAUNCH = 7, 8  # fac_debug_resunit_lanes modes of an encoder unit
# (C, T) of the first two encoder stages at the bench length (4 s at 24 kHz, after the stride-2 down-conv)
ENC_FUSED = ((64, 96000), (128, 48000))


def _plan(L, C, K, dil, T, mode):
    out = (ctypes.c_int * 8)()
    rc = L.fac_debug_tc_plan(C, C, K, dil, 1, T, mode, 0, out)
    return rc, dict(zip(KEYS, list(out)))


@pytest.mark.parametrize("dil", [1, 3, 9])
@pytest.mark.parametrize("C,T", ENC_FUSED)
def test_fused_unit_plan_keeps_two_ctas_and_the_blobs_n(C, T, dil, built_lib):
    """The fused plan fits two CTAs per SM and has N = C, the N both unfused weight blobs were laid out for; its GEMM 1
    runs the unfused conv7's tile (rows, warpgroup split, promotion window)."""
    from facodec_b200 import _lib
    L = _lib.load()
    rc, f = _plan(L, C, 7, dil, T, FUSED_UNIT)
    assert rc == 0, (C, dil)
    rc7, p7 = _plan(L, C, 7, dil, T, PLAIN)
    rc1, p1 = _plan(L, C, 1, 1, T, PLAIN)
    assert rc7 == 0 and rc1 == 0
    assert f["smem"] <= SMEM_CAP2, f
    assert f["N"] == C == p7["N"] == p1["N"], (f, p7, p1)
    for k in ("MT", "rows", "nchunk", "Rpad", "promote_every"):
        assert f[k] == p7[k], (k, f, p7)
    assert p1["nchunk"] <= 48                     # the 1x1 is one promotion window in both routes


def test_c128_fused_plan_costs_no_shared_memory_over_its_conv7(built_lib):
    """At C = 128 the GEMM-2 operand takes the place of the master accumulator (both 32 KB): the fused unit needs no more
    shared memory than the unfused conv7 (105 856 B at d = 9)."""
    from facodec_b200 import _lib
    L = _lib.load()
    for dil in (1, 3, 9):
        _, f = _plan(L, 128, 7, dil, 48000, FUSED_UNIT)
        _, p7 = _plan(L, 128, 7, dil, 48000, PLAIN)
        assert f["smem"] == p7["smem"], (dil, f, p7)
    assert _plan(L, 128, 7, 9, 48000, FUSED_UNIT)[1]["smem"] == 105856


@pytest.mark.parametrize("C,T", [(256, 19200), (512, 3840), (32, 96000)])
def test_fused_unit_plan_refused_where_it_cannot_keep_two_ctas(C, T, built_lib):
    """C >= 256 would need NW = 128 promoted accumulators (one CTA per SM), and only NW = 64 is compiled: those units
    keep their two launches."""
    from facodec_b200 import _lib
    L = _lib.load()
    for dil in (1, 3, 9):
        assert _plan(L, C, 7, dil, T, FUSED_UNIT)[0] == FAC_ERR_UNSUPPORTED, (C, dil)


# ---- GPU --------------------------------------------------------------------------------------------------------------

def _engine():
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    return e


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _bits(t):
    return t.contiguous().view(torch.int32)


def _unit(C, dil, causal, T):
    """Weights of one unit, a ragged batch (lanes of T, 1, short, tile-edge and odd lengths; x NaN past each lane's end)
    and each lane's fp64 reference."""
    from oracle import facodec_oracle as O
    gen = torch.Generator().manual_seed(C * 1000 + dil * 10 + int(causal) + T)
    lens = [T, 1, 13, 64, 129, T - 1, 200]
    lens = [L for L in lens if 1 <= L <= T]
    B = len(lens)
    x = torch.randn(B, C, T, generator=gen) * 0.5
    for b, L in enumerate(lens):
        x[b, :, L:] = float("nan")
    w = dict(w7=torch.randn(C, C, 7, generator=gen) / math.sqrt(C * 7), b7=torch.randn(C, generator=gen) * 0.1,
             w1=torch.randn(C, C, 1, generator=gen) / math.sqrt(C), b1=torch.randn(C, generator=gen) * 0.1,
             a1=torch.rand(C, generator=gen) + 0.5, a2=torch.rand(C, generator=gen) + 0.5)
    sd = {"u.block.0.alpha": w["a1"].view(1, C, 1), "u.block.1.conv.conv.weight": w["w7"], "u.block.1.conv.conv.bias": w["b7"],
          "u.block.2.alpha": w["a2"].view(1, C, 1), "u.block.3.conv.conv.weight": w["w1"], "u.block.3.conv.conv.bias": w["b1"]}
    sd = {k: v.double() for k, v in sd.items()}
    refs = [O.residual_unit(x[b:b + 1, :, :L].double(), sd, "u", dil, causal=causal)[0] for b, L in enumerate(lens)]
    return lens, x, w, refs


def _run(e, w, x_cl, C, dil, mode, causal, lens):
    B, T = x_cl.shape[0], x_cl.shape[1]
    y = torch.full((B, T, C), float("nan"), device="cuda")
    rc = e.L.fac_debug_resunit_lanes(e.handle, _p(x_cl), _p(w["w7"].contiguous()), _p(w["b7"]), _p(w["w1"].contiguous()),
                                     _p(w["b1"]), _p(w["a1"]), _p(w["a2"]), B, T, C, dil, mode, int(causal),
                                     (ctypes.c_int * B)(*lens), _p(y), None)
    assert rc == 0, e.L.fac_last_error(e.handle)
    return y.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("T", [300, 1111])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dil", [1, 3, 9])
@pytest.mark.parametrize("C", [64, 128])
def test_fused_unit_equals_two_launches(C, dil, causal, T, built_lib):
    """One fused launch against the two promoted launches of the same unit, into NaN-filled outputs: every row of every
    lane bit-equal and finite (written).  T is no multiple of the 128- or 64-row tile; C = 128 sums its conv7 in two
    promotion windows.  Both are also held to fp64 at the 3xTF32 unit bound."""
    e = _engine()
    lens, x, w, refs = _unit(C, dil, causal, T)
    x_cl = x.transpose(1, 2).contiguous().cuda()
    y2 = _run(e, w, x_cl, C, dil, TWO_LAUNCHES, causal, lens)
    y1 = _run(e, w, x_cl, C, dil, ONE_LAUNCH, causal, lens)
    for b, L in enumerate(lens):
        assert torch.isfinite(y1[b, :L]).all(), f"lane {b} (L = {L}): a row was not written"
        assert torch.equal(_bits(y1[b, :L]), _bits(y2[b, :L])), f"lane {b} (L = {L}): fused differs from two launches"
        ref = refs[b]
        err = (y1[b, :L].t().double() - ref).abs().max().item()
        assert err <= 8e-5 * max(ref.abs().max().item(), 1.0), f"lane {b} (L = {L}): max err {err}"


def _codec():
    import facodec_b200 as fb
    from facodec_b200 import synth
    sds = synth.synth_state_dicts(0)
    model = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        model[k].load_state_dict(sds[k])
        model[k].eval()
    return fb.Codec(model), synth


def _encode_tapped(codec, x, lengths, fuse):
    B, _, T = x.shape
    eng = codec.engine
    taps, t, ch = {}, T, 64
    for i, s in enumerate((2, 5, 5, 6)):
        for j in range(3):
            taps[f"enc_block{i + 1}.res{j}"] = torch.full((B, t, ch), float("nan"), device="cuda")
        t, ch = -(-t // s), 2 * ch
    eng.set_option("fuse_resunit", fuse)
    try:
        for n, buf in taps.items():
            eng.L.fac_debug_tap(eng.handle, n.encode(), _p(buf), buf.numel())
        codes, timbre = codec.encode(x, n_c=2, lengths=lengths)
        torch.cuda.synchronize()
        launches = codec.launch_count()
    finally:
        for n in taps:
            eng.L.fac_debug_tap(eng.handle, n.encode(), None, 0)
        eng.set_option("fuse_resunit", 1)
    return codes, timbre, taps, launches


@pytest.mark.gpu
@pytest.mark.parametrize("lengths", [None, (9600, 4321, 7777)])
def test_codec_encode_fused_units_bit_identical(lengths, built_lib):
    """Codec.encode with the encoder's C = 64 and 128 units fused (fuse_resunit = 1) against two launches each
    (fuse_resunit = 0): codes, timbre and every unit's output tap bit-identical, and exactly 6 launches fewer."""
    codec, synth = _codec()
    x = synth.synth_waves(3, 9600, seed=5).contiguous().cuda()
    c0, t0, taps0, n0 = _encode_tapped(codec, x, lengths, 0)
    c1, t1, taps1, n1 = _encode_tapped(codec, x, lengths, 1)
    for a, b in zip(c0, c1):
        assert torch.equal(a, b), "codes differ"
    assert torch.equal(_bits(t0), _bits(t1)), "timbre differs"
    for n in taps0:
        assert torch.equal(_bits(taps0[n]), _bits(taps1[n])), f"{n} differs"
        assert lengths is not None or torch.isfinite(taps1[n]).all(), f"{n}: tap not written"
    assert n0 - n1 == 6, (n0, n1)
