"""GPU: the conv kernels on ragged batches and in the non-causal geometry, lane by lane against float64.

A ragged batch gives every conv kernel a per-lane length (ConvParams::lane_len / TcConvParams::lane_len): lane b pads its
own first L_b rows (PadMap::lane).  fac_debug_conv_lanes / fac_debug_resunit_lanes run one layer so, at the channel
counts, kernel sizes and paddings of every call site that passes lengths (engine.cu: the encoder, the codec decoder and
the redecoder's non-causal one, the StyleEncoder's GLU convs, both WaveNets, the FMA-path mel DFT).  Each lane is held to:

* the oracle's own layer in float64 on the lane's own sequence x[b, :, :L_b], on the lane's own output rows, within the
  precision class's bound of test_gpu_kernels.py relative to the lane's own scale;
* no read past its end: its input rows t >= L_b are NaN, and every output row of the batch (the lanes' tails included)
  must come out finite -- a unit adds x to every row, so there the tails must come out NaN instead;
* the ragged contract: its rows equal, bit for bit, the same hook on that lane alone (B = 1, Tin = L_b, that length's
  own pads).

The batch's pads come from Tin by the engine's rule (SConv1d's extra padding), as the product passes them."""
import ctypes
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

FAC_ERR_INVALID, FAC_ERR_UNSUPPORTED = -1, -4
NAN = float("nan")
# per-class bounds of test_gpu_kernels.py: path -1 = the fp32 FMA kernels, 0..5 = the tensor-core classes of
# fac_debug_conv_tc; the unit modes as test_residual_unit_modes
CONV_TOL = {-1: 2e-5, 0: 6e-5, 1: 4e-6, 2: 2e-4, 3: 4e-6, 4: 4e-6, 5: 2e-3}
UNIT_TOL = {0: 2e-5, 1: 8e-5, 2: 8e-5, 3: 3e-4, 4: 3e-4, 5: 2e-3, 6: 2e-3}


def _engine(occ2=0):
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    e.set_option("tc_occ2_maxn", occ2)
    return e


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _ints(v):
    return (ctypes.c_int * len(v))(*v) if v is not None else None


def _seed(name):
    return zlib.crc32(name.encode()) % 100000


def lane_lengths(Tin, max_pad, tiles, B=None, seed=0):
    """Tin, both sides of pad1d's short-input branch (max_pad, max_pad + 1), 1, lanes ending on the last and on the first
    row of a time tile (tiles), Tin - 1; with B, random lengths in [1, Tin] up to B lanes.  Shuffled: not sorted."""
    lens = []
    for L in [Tin, max_pad, max_pad + 1, 1] + list(tiles) + [Tin - 1]:
        if 1 <= L <= Tin and L not in lens:
            lens.append(L)
    g = torch.Generator().manual_seed(seed)
    while B is not None and len(lens) < B:
        lens.append(int(torch.randint(1, Tin + 1, (1,), generator=g)))
    lens = [lens[i] for i in torch.randperm(len(lens), generator=g).tolist()]
    assert len(lens) >= 5 and lens != sorted(lens) and lens != sorted(lens, reverse=True)
    return lens


def sconv_pads(T, k_eff, stride, causal):
    """SConv1d's padding of a T-row input (encodec.py:212-228 with get_extra_padding_for_conv1d): (left, right, Tout)."""
    from oracle import facodec_oracle as O
    total = k_eff - stride
    extra = O._extra_padding(T, k_eff, stride, total)
    pl = total if causal else total - total // 2
    pr = (0 if causal else total // 2) + extra
    return pl, pr, (T + pl + pr - k_eff) // stride + 1


# Every conv call site that passes lane lengths, at the product's geometry (pack_encoder, pack_decoder_into,
# pack_redecoder, pack_quantizer; synth.py's shapes).  kind: sconv = SConv1d (reflect), glu = Conv1dGLU's conv (zero pad
# 2 / 2), up = SConvTranspose1d(2s, s) in its conv form (fac_debug_convtr_pack: 2 taps causal, 3 non-causal, zero pad),
# mel = the FMA-path STFT as a conv (reflect 600 / 600).  step: input rows per output row (the tile lengths scale by it).
# tiles (extra): lane ends about the cin1 kernel's 256-row tile.
CONVS = {
    "enc.conv0": dict(kind="sconv", Cin=1, Cout=64, K=7, stride=1, causal=True, snake=0, Tin=600, tiles=(256, 257, 512, 513)),
    "enc.down.s2": dict(kind="sconv", Cin=64, Cout=128, K=4, stride=2, causal=True, snake=1, Tin=300),
    "enc.down.s5a": dict(kind="sconv", Cin=128, Cout=256, K=10, stride=5, causal=True, snake=1, Tin=700),
    "enc.down.s5b": dict(kind="sconv", Cin=256, Cout=512, K=10, stride=5, causal=True, snake=1, Tin=700),
    "enc.down.s6": dict(kind="sconv", Cin=512, Cout=1024, K=12, stride=6, causal=True, snake=1, Tin=800),
    "enc.conv_out": dict(kind="sconv", Cin=1024, Cout=1024, K=3, stride=1, causal=True, snake=1, Tin=140),
    "dec.conv0.causal": dict(kind="sconv", Cin=1024, Cout=1536, K=7, stride=1, causal=True, snake=0, Tin=140),
    "dec.conv0.noncausal": dict(kind="sconv", Cin=1024, Cout=1536, K=7, stride=1, causal=False, snake=0, Tin=140),
    "dec.up.s6.causal": dict(kind="up", Cin=1536, Cout=768, stride=6, causal=True, Tin=130),
    "dec.up.s6.noncausal": dict(kind="up", Cin=1536, Cout=768, stride=6, causal=False, Tin=130),
    "dec.up.s5a.causal": dict(kind="up", Cin=768, Cout=384, stride=5, causal=True, Tin=140),
    "dec.up.s5a.noncausal": dict(kind="up", Cin=768, Cout=384, stride=5, causal=False, Tin=140),
    "dec.up.s5b.causal": dict(kind="up", Cin=384, Cout=192, stride=5, causal=True, Tin=160),
    "dec.up.s5b.noncausal": dict(kind="up", Cin=384, Cout=192, stride=5, causal=False, Tin=160),
    "dec.up.s2.causal": dict(kind="up", Cin=192, Cout=96, stride=2, causal=True, Tin=200),
    "dec.up.s2.noncausal": dict(kind="up", Cin=192, Cout=96, stride=2, causal=False, Tin=200),
    "dec.conv_out.causal": dict(kind="sconv", Cin=96, Cout=1, K=7, stride=1, causal=True, snake=1, act=1, Tin=300),
    "dec.conv_out.noncausal": dict(kind="sconv", Cin=96, Cout=1, K=7, stride=1, causal=False, snake=1, act=1, Tin=300),
    "se.glu": dict(kind="glu", Cin=512, Cout=1024, K=5, Tin=140),
    "wn.in": dict(kind="sconv", Cin=256, Cout=512, K=5, stride=1, causal=True, snake=0, Tin=200),
    "wn.rs": dict(kind="sconv", Cin=256, Cout=512, K=1, stride=1, causal=True, snake=0, Tin=200),
    "red.in": dict(kind="sconv", Cin=512, Cout=1024, K=5, stride=1, causal=False, snake=0, Tin=140),
    "red.in.b35": dict(kind="sconv", Cin=512, Cout=1024, K=5, stride=1, causal=False, snake=0, Tin=140, B=35),
    "red.rs": dict(kind="sconv", Cin=512, Cout=1024, K=1, stride=1, causal=False, snake=0, Tin=140),
    "mel.dft": dict(kind="mel", Cin=1, Cout=2050, K=1200, stride=300, Tin=39000,
                    tiles=(63 * 300 + 150, 64 * 300 + 7, 127 * 300 + 13, 128 * 300 + 1)),
}


def _tc_eligible(g):
    return g["Cin"] % 16 == 0 and g["Cout"] % 16 == 0


def _layer(g):
    """(Cin, Cout, K, stride) of the conv the hook runs, and the layer's max_pad (pad1d's short-input threshold)."""
    if g["kind"] == "up":
        taps = 2 if g["causal"] else 3
        return g["Cin"], g["stride"] * g["Cout"], taps, 1, 1
    if g["kind"] == "glu":
        return g["Cin"], g["Cout"], g["K"], 1, 2
    if g["kind"] == "mel":
        return g["Cin"], g["Cout"], g["K"], g["stride"], 600
    pl, pr, _ = sconv_pads(g["Tin"], g["K"], g["stride"], g["causal"])
    return g["Cin"], g["Cout"], g["K"], g["stride"], max(pl, pr)


def _pads(g, T):
    """(pad_left, pad_right, reflect, Tout) the product passes for a T-row input of layer g."""
    if g["kind"] == "up":
        return 1, 0 if g["causal"] else 1, 0, T
    if g["kind"] == "glu":
        return 2, 2, 0, T
    if g["kind"] == "mel":
        return 600, 600, 1, (T + 1200 - g["K"]) // g["stride"] + 1
    pl, pr, Tout = sconv_pads(T, g["K"], g["stride"], g["causal"])
    return pl, pr, 1, Tout


_CASES = {}


def _conv_case(name):
    """Weights, the poisoned batch and each lane's float64 reference of layer `name` (built once per module)."""
    if name in _CASES:
        return _CASES[name]
    from facodec_b200 import _lib
    from oracle import facodec_oracle as O
    g = CONVS[name]
    gen = torch.Generator().manual_seed(_seed(name))
    Cin, Cf, Kf, sf, max_pad = _layer(g)
    step = g.get("stride", 1) if g["kind"] == "sconv" else 1
    tiles = [64 * step, 64 * step + 1, 128 * step, 128 * step + 1] + list(g.get("tiles", ()))
    if g["kind"] == "mel":
        tiles = list(g["tiles"])
    lens = lane_lengths(g["Tin"], max_pad, tiles, B=g.get("B"), seed=_seed(name))
    B, Tin = len(lens), g["Tin"]
    x = torch.randn(B, Cin, Tin, generator=gen) * 0.5
    for b, L in enumerate(lens):
        x[b, :, L:] = NAN                          # poison: no kernel may read a row at or past the lane's end
    ia = torch.rand(Cin, generator=gen) + 0.5 if g.get("snake") or g["kind"] == "up" else None
    c = dict(lens=lens, x=x, ia=ia, act=g.get("act", 0), layer=(Cin, Cf, Kf, sf))
    if g["kind"] == "up":
        s, Cout = g["stride"], g["Cout"]
        wt = torch.randn(Cin, Cout, 2 * s, generator=gen) / math.sqrt(Cin * 2)
        bt = torch.randn(Cout, generator=gen) * 0.1
        L = _lib.load()
        taps = Kf
        pk = torch.zeros(taps * Cin * Cf)
        assert L.fac_debug_convtr_pack(_p(wt.contiguous()), Cin, Cout, s, int(g["causal"]), _p(pk), pk.numel()) == pk.numel()
        c["w"] = pk.view(taps, Cin, Cf).permute(2, 1, 0).contiguous()          # conv1d weight [s*Cout][Cin][taps]
        c["b"] = bt.repeat(s)                                                     # channel r*Cout + co: phase r
        sd = {"c.weight": wt.double(), "c.bias": bt.double()}
    else:
        c["w"] = torch.randn(Cf, Cin, Kf, generator=gen) / math.sqrt(Cin * Kf)
        c["b"] = torch.randn(Cf, generator=gen) * 0.1 if g["kind"] != "mel" else None
        sd = {"c.weight": c["w"].double(), "c.bias": c["b"].double() if c["b"] is not None else None}
    refs = []
    for b, L in enumerate(lens):
        xb = x[b:b + 1, :, :L].double()
        if ia is not None:
            xb = O.snake(xb, ia.double().view(1, -1, 1))
        if g["kind"] == "up":
            r = O.sconvtr1d(xb, sd, "c", g["stride"], causal=g["causal"])            # [1, Cout, s * L]
        elif g["kind"] == "glu":
            r = F.conv1d(F.pad(xb, (2, 2)), sd["c.weight"], sd["c.bias"])
        elif g["kind"] == "mel":
            r = F.conv1d(O._pad1d_reflect(xb, 600, 600), sd["c.weight"], None, stride=g["stride"])
        else:
            r = O.sconv1d(xb, sd, "c", stride=g["stride"], causal=g["causal"])
        if c["act"] == 1:
            r = torch.tanh(r)
        refs.append(r[0])
    c["refs"] = refs
    _CASES[name] = c
    return c


def _run_conv(e, g, c, x_cl, lens, T, path):
    """fac_debug_conv_lanes on channels-last x_cl [B][T][Cin]; returns (status, y [B][Tout][Cf] on the host)."""
    Cin, Cf, Kf, sf = c["layer"]
    pl, pr, reflect, Tout = _pads(g, T)
    B = x_cl.shape[0]
    y = torch.full((B, Tout, Cf), NAN, device="cuda")
    rc = e.L.fac_debug_conv_lanes(e.handle, _p(x_cl), _p(c["w"]), _p(c["b"]), B, T, Cin, Cf, Kf, 1, sf, pl, pr, reflect,
                                  _p(c["ia"]), None, c["act"], None, _p(y), Tout, path, _ints(lens), None)
    return rc, y.cpu()


def _lane_rows(g, y, b, n):
    """Lane b's first n output rows of the hook's y, as the reference lays them out: [Cout, n]."""
    if g["kind"] == "up":                      # phase-major channels: frame t, channel r*Cout + co = sample t*s + r
        s, Cout = g["stride"], g["Cout"]
        return y[b, :n // s].reshape(n, Cout).t()
    return y[b, :n].t()


CONV_PARAMS = [(n, p, o) for n in CONVS for p in ([-1] + ([0, 1, 2, 3, 4, 5] if _tc_eligible(CONVS[n]) else []))
               for o in ((0,) if p == -1 else (0, 256)) if not (o and p in (1, 3, 4))]


@pytest.mark.parametrize("name,path,occ2", CONV_PARAMS)
def test_conv_lanes_vs_fp64(name, path, occ2, built_lib):
    """One ragged layer of every lane-passing call site, through the FMA kernels (path -1: cin1 / cout1 / generic, as
    tensor_cores = 0 runs ragged batches) and every tensor-core class (path 0..5, occ2 = tiles planned for two CTAs per
    SM; the promoted classes have a single residency plan)."""
    g = CONVS[name]
    c = _conv_case(name)
    e = _engine(occ2)
    lens, Tin = c["lens"], g["Tin"]
    x_cl = c["x"].transpose(1, 2).contiguous().cuda()
    rc, y = _run_conv(e, g, c, x_cl, lens, Tin, path)
    if path >= 0 and rc == FAC_ERR_UNSUPPORTED:
        pytest.skip(f"class {path} does not plan this layer: {e.L.fac_last_error(e.handle)}")
    assert rc == 0, e.L.fac_last_error(e.handle)
    assert torch.isfinite(y).all(), "a lane read a row past its end, or a row of y was not written"
    tol = CONV_TOL[path]
    for b, L in enumerate(lens):
        ref = c["refs"][b]
        n = ref.shape[-1]
        got = _lane_rows(g, y, b, n)
        err = (got.double() - ref).abs().max().item()
        scale = ref.abs().max().item()
        print(f"LANES {name} path={path} occ2={occ2} L={L} rows={n} maxerr={err:.3e} scale={scale:.3f}")
        assert err <= tol * max(scale, 1.0), f"lane {b} (L = {L}): max err {err} (scale {scale})"
        # the ragged contract: the lane alone, with its own length's pads
        rc1, y1 = _run_conv(e, g, c, x_cl[b:b + 1, :L].contiguous(), None, L, path)
        assert rc1 == 0, e.L.fac_last_error(e.handle)
        assert torch.equal(_lane_rows(g, y1, 0, n), got), f"lane {b} (L = {L}) differs from its B = 1 call"


# ResidualUnits of every stage: the encoder's (causal, C = 64..512) and both decoders' (C = 768..96, causal for the codec,
# non-causal for the redecoder).  (C, dil, causal, T)
UNITS = ([(C, d, True, T) for C, T in ((64, 300), (128, 300), (256, 200), (512, 140)) for d in (1, 3, 9)] +
         [(C, d, cz, T) for C, T in ((768, 130), (384, 160), (192, 200), (96, 300)) for d in (1, 9) for cz in (True, False)])
_UNIT_CASES = {}


def _unit_case(C, dil, causal, T):
    key = (C, dil, causal, T)
    if key in _UNIT_CASES:
        return _UNIT_CASES[key]
    from oracle import facodec_oracle as O
    gen = torch.Generator().manual_seed(C * 100 + dil * 10 + int(causal))
    k_eff = 6 * dil + 1
    max_pad = k_eff - 1 if causal else (k_eff - 1) - (k_eff - 1) // 2
    lens = lane_lengths(T, max_pad, (64, 65, 128, 129), seed=C + dil)
    B = len(lens)
    x = torch.randn(B, C, T, generator=gen) * 0.5
    for b, L in enumerate(lens):
        x[b, :, L:] = NAN
    w = dict(w7=torch.randn(C, C, 7, generator=gen) / math.sqrt(C * 7), b7=torch.randn(C, generator=gen) * 0.1,
             w1=torch.randn(C, C, 1, generator=gen) / math.sqrt(C), b1=torch.randn(C, generator=gen) * 0.1,
             a1=torch.rand(C, generator=gen) + 0.5, a2=torch.rand(C, generator=gen) + 0.5)
    sd = {"u.block.0.alpha": w["a1"].view(1, C, 1), "u.block.1.conv.conv.weight": w["w7"], "u.block.1.conv.conv.bias": w["b7"],
          "u.block.2.alpha": w["a2"].view(1, C, 1), "u.block.3.conv.conv.weight": w["w1"], "u.block.3.conv.conv.bias": w["b1"]}
    sd = {k: v.double() for k, v in sd.items()}
    refs = [O.residual_unit(x[b:b + 1, :, :L].double(), sd, "u", dil, causal=causal)[0] for b, L in enumerate(lens)]
    c = dict(lens=lens, x=x, w=w, refs=refs)
    _UNIT_CASES[key] = c
    return c


def run_unit(e, w, x_cl, C, dil, mode, causal, lens, fill=NAN):
    B, T = x_cl.shape[0], x_cl.shape[1]
    y = torch.full((B, T, C), fill, device="cuda")
    rc = e.L.fac_debug_resunit_lanes(e.handle, _p(x_cl), _p(w["w7"].contiguous()), _p(w["b7"]), _p(w["w1"].contiguous()),
                                     _p(w["b1"]), _p(w["a1"]), _p(w["a2"]), B, T, C, dil, mode, int(causal), _ints(lens),
                                     _p(y), None)
    return rc, y.cpu()


@pytest.mark.parametrize("occ2", [0, 256])
@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4, 5, 6])
@pytest.mark.parametrize("C,dil,causal,T", UNITS)
def test_residual_unit_lanes_vs_fp64(C, dil, causal, T, mode, occ2, built_lib):
    """A ragged ResidualUnit in every mode of fac_debug_resunit (0 FMA, 1 / 3 / 5 two tensor-core launches, 2 / 4 / 6
    the fused launch).  The unit adds x to every row, so a lane's tail rows (x = NaN there) must come out NaN: y starts
    finite, and a tail row left as it was is a row the kernel never wrote."""
    if occ2 and mode == 0:
        pytest.skip("fp32 FMA path has no residency option")
    c = _unit_case(C, dil, causal, T)
    e = _engine(occ2)
    lens = c["lens"]
    x_cl = c["x"].transpose(1, 2).contiguous().cuda()
    rc, y = run_unit(e, c["w"], x_cl, C, dil, mode, causal, lens, fill=7.0)
    if (mode == 2 and C > 128) or (mode in (4, 6) and C > 256):
        # the fused launch holds every channel in one CTA tile: up to C = 128 with the tf32 split, 256 with the 16-bit
        # ones (test_residual_unit_modes); the wider units run as two launches (modes 1 / 3 / 5)
        assert rc == FAC_ERR_UNSUPPORTED
        return
    assert rc == 0, e.L.fac_last_error(e.handle)
    tol = UNIT_TOL[mode]
    for b, L in enumerate(lens):
        got = y[b, :L].t()
        assert torch.isfinite(got).all(), f"lane {b} (L = {L}) read a row past its end"
        assert torch.isnan(y[b, L:]).all(), f"lane {b} (L = {L}): a tail row was not written"
        ref = c["refs"][b]
        err = (got.double() - ref).abs().max().item()
        scale = ref.abs().max().item()
        print(f"UNITLANES C={C} d={dil} causal={causal} mode={mode} occ2={occ2} L={L} maxerr={err:.3e} scale={scale:.3f}")
        assert err <= tol * max(scale, 1.0), f"lane {b} (L = {L}): max err {err} (scale {scale})"
        rc1, y1 = run_unit(e, c["w"], x_cl[b:b + 1, :L].contiguous(), C, dil, mode, causal, None)
        assert rc1 == 0, e.L.fac_last_error(e.handle)
        assert torch.equal(y1[0].t(), got), f"lane {b} (L = {L}) differs from its B = 1 call"


def test_lane_lengths_out_of_range_rejected(built_lib):
    """A lane length of 0 or Tin + 1 is refused before anything is launched: FAC_ERR_INVALID, y untouched."""
    e = _engine()
    B, T, C = 3, 40, 64
    x = torch.randn(B, T, C, device="cuda")
    w = torch.randn(C, C, 7) / math.sqrt(C * 7)
    b = torch.zeros(C)
    for bad in (0, T + 1):
        lens = [T, bad, 5]
        for path in (-1, 0):
            y = torch.full((B, T, C), 3.0, device="cuda")
            rc = e.L.fac_debug_conv_lanes(e.handle, _p(x), _p(w), _p(b), B, T, C, C, 7, 1, 1, 6, 0, 1, None, None, 0, None,
                                          _p(y), T, path, _ints(lens), None)
            assert rc == FAC_ERR_INVALID and b"lane lengths" in e.L.fac_last_error(e.handle)
            assert (y == 3.0).all()
        y = torch.full((B, T, C), 3.0, device="cuda")
        wu = dict(w7=w, b7=b, w1=torch.randn(C, C, 1) / 8, b1=b, a1=torch.ones(C), a2=torch.ones(C))
        rc, yu = run_unit(e, wu, x, C, 1, 4, 0, lens, fill=3.0)
        assert rc == FAC_ERR_INVALID and b"lane lengths" in e.L.fac_last_error(e.handle)
        assert (yu == 3.0).all()


@pytest.mark.parametrize("path", [-1, 0, 1, 2, 3, 4, 5])
def test_snake_large_argument(path, built_lib):
    """Snake past |alpha x| = 4096, where sin2_f / snake4 leave the polynomial for sinf() (inlined in the setmaxnreg
    kernels; classes 2 and 5 take snake4_mufu, which has no range check).  A 1x1 conv 64 -> 64 with in- and out-Snake
    whose weights are near the identity, so the out-Snake sees large arguments too.  Each row is held to its class's
    bound relative to its own scale, so the large rows cannot hide an error in the others, nor the others in them: a
    dropped sin^2 term is up to 1 / alpha on a row of scale ~ 4400 / alpha."""
    from test_gpu_kernels import ref_conv
    C, T = 64, 200
    e = _engine()
    gen = torch.Generator().manual_seed(4096)
    ia = torch.rand(C, generator=gen) * 0.4 + 0.8
    oa = torch.rand(C, generator=gen) * 0.4 + 0.8
    x = torch.randn(1, C, T, generator=gen) * 0.5
    sign = lambda: torch.where(torch.rand(C, generator=gen) < 0.5, -1.0, 1.0)
    for t in (10, 11, 64, 65, 127, 150):       # |alpha x| just above the threshold
        x[0, :, t] = sign() * (4097.0 + 200.0 * torch.rand(C, generator=gen)) / ia
    for t in (30, 140):                        # up to 5e4: the 2^12 pi reduction range and past it, inside fp16's range
        x[0, :, t] = sign() * torch.exp(torch.empty(C).uniform_(math.log(4097.0), math.log(5e4), generator=gen)) / ia
    w = torch.eye(C).view(C, C, 1) + torch.randn(C, C, 1, generator=gen) * 0.01
    b = torch.randn(C, generator=gen) * 0.1
    ref = ref_conv(x, w, b, 1, 1, 0, 0, 0, ia, oa, 0, None)[0]                # [C, T] float64
    xd = x.transpose(1, 2).contiguous().cuda()
    yd = torch.full((1, T, C), NAN, device="cuda")
    rc = e.L.fac_debug_conv_lanes(e.handle, _p(xd), _p(w.contiguous()), _p(b), 1, T, C, C, 1, 1, 1, 0, 0, 0, _p(ia), _p(oa),
                                  0, None, _p(yd), T, path, None, None)
    assert rc == 0, e.L.fac_last_error(e.handle)
    y = yd.cpu()[0].t().double()
    assert torch.isfinite(y).all()
    err = (y - ref).abs().amax(0)
    scale = ref.abs().amax(0).clamp(min=1.0)
    worst = int((err / scale).argmax())
    print(f"SNAKE path={path} worst row {worst}: err {err[worst]:.3e} scale {scale[worst]:.3e}")
    assert (err <= CONV_TOL[path] * scale).all(), f"row {worst}: max err {err[worst]} (scale {scale[worst]})"
