"""The codec encoder and decoder, layer by layer, against a plain float64 restatement, on every precision route.

Each step between two of the engine's debug taps is one layer or one ResidualUnit:

  encoder  enc_conv0 (conv0)  enc_block<i>.res<j> (unit j of EncoderBlock i)  enc_block<i> (Snake + strided down-conv)
           enc_lstm (SLSTM)  z (Snake + conv_out, the Encoder output)
  decoder  dec_conv0  dec_lstm (codec only)  dec_block<i>.up (Snake + up-conv)  dec_block<i>.res<j>
           y (Snake + conv_out + tanh, the Decoder output)

Teacher forcing: each step's input is the GPU's own tap of the step before it, so every comparison measures that one
step's error, not an error carried in from earlier layers.  The tap buffers are NaN before the call, and every step's
output must come out finite.  This checks what the engine dispatches when it runs its own encoder and decoder: the
precision class run_conv picks for each layer, the short-chain 1x1 convs of the 64- and 128-channel encoder stages,
the fused or two-launch ResidualUnit, the LSTM class, weight-norm folding and packing of a real state dict (the
phase-major transposed convs included), and the three rotating stage buffers.

Reference (this file, from the oracle's own primitives O.snake, O.sconv1d, O.sconvtr1d, O._wn_weight and
test_gpu_lstm.slstm_ref).  A precision class is modelled by the rounding of both operands of each conv: exact, "fp16"
(one pass over fp16-rounded operands) or "bf16x3" (bf16 hi = rn(v), lo = rn(v - hi), products hh + hl + lh), with
test_gpu_lstm's f16_rn / bf16_split.  Rounding is elementwise and commutes with padding and unfolding, so a class's
products are the oracle's conv of the rounded operands (three convs for bf16x3, as test_gpu_lstm._mm forms them); the
oracle's conv then covers the dilated, strided, transposed and non-causal layers, which test_gpu_wavenet._sconv (stride 1,
no dilation) does not, with no restatement of the engine's packing.  CPU tests check the exact chain equals
O.encoder_forward / O.decoder_forward and their taps in float64.  On the GPU the references run in float64 (y64), with a
class's rounding (y_cls), and in float32 (y32) with TF32 off (cuBLAS and cuDNN; see _fp32 for why the convs of y32
stay on cuDNN).

Bars (factors below, floor C relative to max|y64|):
* Encoder steps, fp32-grade because they feed the bit-exact VQ argmin: max|y - y64| <= F max|y32 - y64| + C max|y64|,
  F = F32 for the FMA kernels and the promoted fp16-pair class, F_TF32X3 with encoder_f16x2 = 0.  Every promoted encoder
  layer runs the promoted kernel (the 1x1 convs of blocks 1 and 2 included, see below).
  Separation: rms(y - y64) <= SEP_ENC rms(y_bf16x3 - y64).  SEP_ENC is 1/2, as test_gpu_wavenet.py uses for the prosody
  branch, not 1/8: from block 2's down-conv on, fp32 accumulation over 1280 - 6144 products is itself within 8x of the
  bf16x3 rounding error, so the fp32 FMA kernels measure rms 0.13 - 0.33 of it there and a 1/8 bar would fail the
  fp32 kernel itself.  A layer on the bf16x3 class measures about 1, so 1/2 still fails it.
* Decoder steps: max|y - y64| <= F_CLS max|y_cls - y64| + C max|y64|, y_cls the emulated class of the route: by default
  the up-convs of blocks 2 - 4 and the units' 1x1 as bf16x3, the units' k = 7 conv as one fp16 pass.  conv0 and block 1's
  up-conv run the promoted fp16-pair class on every tensor-core route and are held to F32 max|y32 - y64|, as conv_out
  (the fp32 FMA kernel) and every step of tensor_cores = 0 are.  decoder_bf16 = 0 (the non-promoted 3xTF32 class, whose
  accumulation truncates) is held to F_TF32X3_TRUNC max|y32 - y64|, as in test_gpu_lstm.py.  decoder_conv7_fp16 = 0 runs
  the units' k = 7 on the non-promoted bf16 hi/lo class, whose accumulation truncates the same way: over block 1's
  5376-long chains that measured 2.6 - 4.4x the bf16x3 rounding model (a bar of F_CLS times the model cannot hold for
  that class), so the units of that route are held to F_TF32X3_TRUNC too, and to the separation below.
  Separation: conv0 and every up-conv rms(y - y64) <= SEP rms(y_fp16 - y64), which fails if that conv runs the
  one-pass fp16 blob; with decoder_conv7_fp16 = 0 and tensor_cores = 0 every unit the same against the unit with its
  k = 7 conv in one fp16 pass.  The decoder SLSTM is held to test_gpu_lstm.check_against_reference's bar of its class.
  A 1x1 conv demoted to one fp16 pass inside an otherwise default unit moves the unit's rms error only about 1.5x, so no
  separation bar is claimed for the 1x1.
* tensor_cores = 1 keeps every encoder layer on the FMA kernels (they are upstream of the VQ): every encoder tap equals
  that of tensor_cores = 0 bit for bit.

test_bars_separate_the_classes shows, on the CPU at the seeds and shapes used, that the separation bars can fail: the
wrong class's rms error is at least 1 / SEP (1 / SEP_ENC) times the right one's (measured: encoder block-2 unit 0
bf16x3 / fp32 17x, decoder conv0 fp16 / bf16x3 66x, decoder block-3 unit 0 fp16 k = 7 / all-bf16x3 43x).

What these tests found, and the product changes they led to (measured on an NVIDIA H100 80GB HBM3, 700 W power limit):
  1. Decoder conv0 (1024 x 7 = 7168 products per output) and block 1's up-conv (1536 x 2) on conv_tc_kernel's bf16
     hi/lo class measured 5 - 6x and 2.4 - 2.9x the max error of the bf16x3 rounding model: the truncating tensor-core
     accumulation over such chains adds error the model leaves out.  Both now take the promoted packing
     (pack_decoder_into).  The later up-convs (<= 768 x 2) measured within the model's bar and keep their class.
  2. The units of encoder blocks 1 and 2, whose 1x1 convs a short-chain probe in run_conv moved to conv_tc_kernel's
     3xTF32 class, measured rms 0.14 - 0.30 of the bf16x3 error, about 2.4x the FMA kernels'.  The probe is removed: those
     1x1 convs run the promoted kernel like every other promoted layer.
With both changes every check is asserted.  Measured over every case: largest err / bar 0.29 (encoder), 0.78 (decoder).
Encoder max error 0.8 - 1.5x the fp32 error on the FMA routes and up to 3.6x on the tensor-core routes (bar 6, 12 with
encoder_f16x2 = 0); rms 0.03 - 0.40 of the bf16x3 error (bar 1/2).  Decoder: conv0 and block 1's up-conv 0.23 - 0.93x
the fp32 error on the tensor-core routes (bar 6); the other steps of the default-class routes 0.3 - 1.9x the emulated
class's max error (bar 2.5), conv0 and the up-convs at rms 0.002 - 0.04 of the one-pass fp16 class (bar 1/8); the units
8 - 17x the fp32 error with decoder_conv7_fp16 = 0 and 6 - 33x with decoder_bf16 = 0 (bar 160).  The file's GPU tests
took 88 s.
"""
import functools

import pytest
import torch

from conftest import GOLDEN_CASES, case_inputs, load_golden, state_dicts
from test_gpu_lstm import bf16_split, check_against_reference, f16_rn, slstm_ref
from test_gpu_wavenet import _rms, _sd_to, _tapped, _threads, redecoder_inputs
from test_gpu_wavenet import _with_options as wavenet_with_options

F32 = 6.0                 # fp32 FMA kernels; the promoted fp16 hi + 2^11-scaled lo class
F_TF32X3 = 12.0           # the promoted 3xTF32 class (encoder_f16x2 = 0)
F_TF32X3_TRUNC = 160.0    # the non-promoted 3xTF32 class (decoder_bf16 = 0), as in test_gpu_lstm.py
F_CLS = 2.5               # factor on the emulated class's error (decoder, tensor-core routes)
SEP = 1.0 / 8             # decoder separation: rms error at most SEP x the one-pass fp16 class's
SEP_ENC = 1.0 / 2         # encoder separation: rms error at most SEP_ENC x the bf16x3 class's
C = 1e-7                  # floor, relative to max|y64|

ENC_RATES, DEC_RATES, DILS = (2, 5, 5, 6), (6, 5, 5, 2), (1, 3, 9)
OPTION_DEFAULTS = {"tensor_cores": 2, "encoder_f16x2": 1, "encoder_tt": 0, "decoder_bf16": 1, "decoder_conv7_fp16": 1,
                   "fuse_resunit": 1, "decoder_lstm_fp16": 1, "tc_occ2_maxn": 0}

# operand rounding per layer kind: conv0, c7 / c1 (a unit's k = 7 and 1x1 convs), down, up, out, ih / rec (SLSTM)
CLASSES = {
    None: {},
    "bf16x3": dict.fromkeys(("conv0", "c7", "c1", "down", "up", "out", "ih", "rec"), "bf16x3"),
    "dec": {"conv0": "bf16x3", "up": "bf16x3", "c7": "fp16", "c1": "bf16x3"},     # the decoder's default classes
    "fp16": {"conv0": "fp16", "up": "fp16", "c7": "fp16", "c1": "bf16x3"},
}
ENC_ROUTES = {"default": ({}, F32), "encoder_tt1": ({"encoder_tt": 1}, F32),
              "encoder_f16x2_0": ({"encoder_f16x2": 0}, F_TF32X3), "tensor_cores1": ({"tensor_cores": 1}, F32),
              "tensor_cores0": ({"tensor_cores": 0}, F32)}
# route -> (options, max bar of the other tensor-core conv steps and of the units: a class of CLASSES (F_CLS x its error)
# or a factor on the fp32 error, LSTM config, whether the units get the separation bar against one fp16 pass)
DEC_ROUTES = {"default": ({}, "dec", "dec", "dec", False),
              "decoder_conv7_fp16_0": ({"decoder_conv7_fp16": 0}, "bf16x3", F_TF32X3_TRUNC, "dec", True),
              "decoder_bf16_0": ({"decoder_bf16": 0}, F_TF32X3_TRUNC, F_TF32X3_TRUNC, "dec_fp32", False),
              "fuse_resunit0": ({"fuse_resunit": 0}, "dec", "dec", "dec", False),
              "fuse_resunit2": ({"fuse_resunit": 2}, "dec", "dec", "dec", False),
              "decoder_lstm_fp16_0": ({"decoder_lstm_fp16": 0}, "dec", "dec", "dec_v1", False),
              "tc_occ2_256": ({"tc_occ2_maxn": 256}, "dec", "dec", "dec", False),
              "tensor_cores0": ({"tensor_cores": 0}, F32, F32, "dec", True)}
REDEC_ROUTES = [r for r in DEC_ROUTES if r != "decoder_lstm_fp16_0"]

# ---------------------------------------------------------------------------------------------------------------------
# float64 restatement, one function per step
# ---------------------------------------------------------------------------------------------------------------------
def _wb(sd, prefix):
    from oracle import facodec_oracle as O
    return O._wn_weight(sd, prefix), sd[prefix + ".bias"]


def conv(x, wb, mode, transposed=False, **kw):
    """O.sconv1d (O.sconvtr1d if transposed) of x [B][C][T] with the folded weight and bias wb, both operands rounded as
    `mode` rounds them (test_gpu_lstm._mm): bf16x3 is the sum of the hh, hl and lh convs, the bias added once."""
    from oracle import facodec_oracle as O
    w, b = wb
    op = O.sconvtr1d if transposed else O.sconv1d
    f = lambda xx, ww, bb: op(xx, {"l.weight": ww, "l.bias": bb}, "l", **kw)
    if mode is None:
        return f(x, w, b)
    if mode == "fp16":
        return f(f16_rn(x), f16_rn(w), b)
    xh, xl = bf16_split(x)
    wh, wl = bf16_split(w)
    z = torch.zeros_like(b)
    return f(xh, wh, b) + f(xh, wl, z) + f(xl, wh, z)


def unit(sd, x, m, p, d, causal=True):
    """ResidualUnit (O.residual_unit) with its k = 7 and 1x1 convs rounded as m["c7"] and m["c1"]."""
    from oracle import facodec_oracle as O
    y = O.snake(x, sd[p + ".block.0.alpha"])
    y = conv(y, _wb(sd, p + ".block.1.conv.conv"), m.get("c7"), dilation=d, causal=causal)
    y = O.snake(y, sd[p + ".block.2.alpha"])
    y = conv(y, _wb(sd, p + ".block.3.conv.conv"), m.get("c1"), causal=causal)
    return x + y


def lstm(sd, x, m, p):
    """SLSTM (O.slstm) on x [B][H][T] through test_gpu_lstm.slstm_ref in x's dtype, rounded as m["ih"] / m["rec"]."""
    ws = [sd[f"{p}.{n}_l{l}"] for l in range(2) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    y = slstm_ref(x.transpose(1, 2), ws, x.dtype, ih=m.get("ih"), rec=m.get("rec"))[0]
    return y.transpose(1, 2)


def snake_conv(sd, x, m, alpha, prefix, kind, **kw):
    from oracle import facodec_oracle as O
    return conv(O.snake(x, sd[alpha]), _wb(sd, prefix), m.get(kind), **kw)


def encoder_steps():
    """[(tap name, kind, fn(sd, x, m))]: Encoder.forward (O.encoder_forward) step by step; x [B][C][T] is the previous
    step's output, m the rounding of CLASSES."""
    steps = [("enc_conv0", "conv0", lambda sd, x, m: conv(x, _wb(sd, "block.0.conv.conv"), m.get("conv0")))]
    for i, s in enumerate(ENC_RATES):
        p = f"block.{i + 1}"
        for j, d in enumerate(DILS):
            steps.append((f"enc_block{i + 1}.res{j}", "unit", functools.partial(_unit_step, p=f"{p}.block.{j}", d=d)))
        steps.append((f"enc_block{i + 1}", "down", functools.partial(snake_conv, alpha=p + ".block.3.alpha",
                                                                    prefix=p + ".block.4.conv.conv", kind="down", stride=s)))
    steps.append(("enc_lstm", "lstm", lambda sd, x, m: lstm(sd, x, m, "block.5.lstm")))
    steps.append(("z", "out", functools.partial(snake_conv, alpha="block.6.alpha", prefix="block.7.conv.conv", kind="out")))
    return steps


def _unit_step(sd, x, m, p, d, causal=True):
    return unit(sd, x, m, p, d, causal)


def decoder_steps(causal=True, with_lstm=True):
    """As encoder_steps for Decoder.forward (O.decoder_forward): the codec's (causal, SLSTM) or the redecoder's."""
    base = 2 if with_lstm else 1
    steps = [("dec_conv0", "conv0", lambda sd, x, m: conv(x, _wb(sd, "model.0.conv.conv"), m.get("conv0"), causal=causal))]
    if with_lstm:
        steps.append(("dec_lstm", "lstm", lambda sd, x, m: lstm(sd, x, m, "model.1.lstm")))
    for i, s in enumerate(DEC_RATES):
        p = f"model.{i + base}"
        steps.append((f"dec_block{i + 1}.up", "up",
                      functools.partial(snake_conv, alpha=p + ".block.0.alpha", prefix=p + ".block.1.convtr.convtr",
                                        kind="up", transposed=True, stride=s, causal=causal)))
        for j, d in enumerate(DILS):
            steps.append((f"dec_block{i + 1}.res{j}", "unit",
                          functools.partial(_unit_step, p=f"{p}.block.{j + 2}", d=d, causal=causal)))
    out = functools.partial(snake_conv, alpha=f"model.{4 + base}.alpha", prefix=f"model.{5 + base}.conv.conv", kind="out",
                            causal=causal)
    steps.append(("y", "out", lambda sd, x, m: torch.tanh(out(sd, x, m))))
    return steps


def _chain(steps, sd, x, m=CLASSES[None]):
    out = {}
    for name, _, fn in steps:
        x = fn(sd, x, m)
        out[name] = x
    return out


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the chained restatement is the oracle; the separation bars can fail
# ---------------------------------------------------------------------------------------------------------------------
def _close(got, ref, what):
    err, scale = (got - ref).abs().max().item(), ref.abs().max().item()
    assert err <= 1e-12 * scale, f"{what}: {err:.3e} vs scale {scale:.3e}"


@pytest.mark.parametrize("B,T", [(2, 1500), (1, 3100)])
def test_encoder_reference_matches_the_oracle(B, T):
    """T = 1500 gives block 4's d = 9 units 30 rows (pad1d's short-input branch); 3100 is not a multiple of 300."""
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    _threads()
    sd = _sd_to(state_dicts(0)["encoder"], torch.float64, "cpu")
    x = synth.synth_waves(B, T, seed=T).double()
    taps = {}
    with torch.no_grad():
        z = O.encoder_forward(sd, x, taps=taps)
        got = _chain(encoder_steps(), sd, x)
    for name, ref in taps.items():
        _close(got[name], ref, name)
    _close(got["z"], z, "z")


@pytest.mark.parametrize("causal,with_lstm,B,Tf", [(True, True, 2, 3), (False, False, 1, 4)])
def test_decoder_reference_matches_the_oracle(causal, with_lstm, B, Tf):
    """The codec's decoder and the redecoder's (non-causal, no SLSTM)."""
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    _threads()
    sds = synth.synth_state_dicts(0) if with_lstm else synth.synth_redecoder_state_dicts(0)
    sd = _sd_to(sds["decoder"], torch.float64, "cpu")
    z = torch.randn(B, 1024, Tf, generator=torch.Generator().manual_seed(Tf), dtype=torch.float64)
    taps = {}
    with torch.no_grad():
        y = O.decoder_forward(sd, z, taps=taps, causal=causal, lstm=2 if with_lstm else 0)
        got = _chain(decoder_steps(causal, with_lstm), sd, z)
    for name, ref in taps.items():
        _close(got[name + ".res2" if name.startswith("dec_block") else name], ref, name)     # a block ends with unit 2
    _close(got["y"], y, "y")


def test_bars_separate_the_classes():
    """On the b2_t7200 fixture's inputs (seed 0), each step's input tapped from the exact chain, the separation bars can
    fail: a step on the wrong class measures at least 1 / SEP (SEP_ENC) times the right class's rms error.
      encoder block-2 unit 0: bf16x3 against fp32 (SEP_ENC);  decoder conv0: one fp16 pass against bf16x3 (SEP);
      decoder block-3 unit 0: k = 7 in one fp16 pass against all-bf16x3 (SEP).
    The margin over 1 / SEP is printed; the fp32 side is the CPU's fp32 conv, whose summation order depends on the CPU."""
    _threads()
    c = GOLDEN_CASES["b2_t7200"]
    sds = state_dicts(c["wseed"])
    x, _ = case_inputs(c)
    zq = torch.from_numpy(load_golden("b2_t7200")["outs"]).double()
    with torch.no_grad():
        sd = _sd_to(sds["encoder"], torch.float64, "cpu")
        sd32 = _sd_to(sds["encoder"], torch.float32, "cpu")
        steps = encoder_steps()
        k = [s[0] for s in steps].index("enc_block2.res0")
        xin = _chain(steps[:k], sd, x.double())["enc_block1"]
        _, _, fn = steps[k]
        y64 = fn(sd, xin, CLASSES[None])
        ratios = {"encoder block-2 unit 0": _rms(fn(sd, xin, CLASSES["bf16x3"]) - y64) /
                  _rms(fn(sd32, xin.float(), CLASSES[None]).double() - y64)}
        sd = _sd_to(sds["decoder"], torch.float64, "cpu")
        steps = decoder_steps()
        y64 = steps[0][2](sd, zq, CLASSES[None])
        ratios["decoder conv0"] = _rms(steps[0][2](sd, zq, CLASSES["fp16"]) - y64) / \
            _rms(steps[0][2](sd, zq, CLASSES["bf16x3"]) - y64)
        k = [s[0] for s in steps].index("dec_block3.res0")
        xin = _chain(steps[:k], sd, zq)["dec_block3.up"]
        fn = steps[k][2]
        y64 = fn(sd, xin, CLASSES[None])
        ratios["decoder block-3 unit 0"] = _rms(fn(sd, xin, CLASSES["fp16"]) - y64) / \
            _rms(fn(sd, xin, CLASSES["bf16x3"]) - y64)
    sep = {"encoder block-2 unit 0": SEP_ENC, "decoder conv0": SEP, "decoder block-3 unit 0": SEP}
    print("SEP " + "  ".join(f"{k}: {v:.1f}x (margin {v * sep[k]:.1f} over 1 / {1 / sep[k]:.0f})" for k, v in ratios.items()))
    for k, v in ratios.items():
        assert v >= 1 / sep[k], f"{k}: the classes are {v:.1f}x apart"


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _with_options(eng, opts, fn):
    return wavenet_with_options(eng, opts, fn, OPTION_DEFAULTS)


def _fp32(fn, *a):
    """fn(*a) in fp32 with TF32 off for cuBLAS and cuDNN.  The convs stay on cuDNN: with cuDNN disabled torch runs them as
    im2col + one cuBLAS GEMM, whose blocked accumulation over the long encoder chains is about 7x more accurate than any
    serial fp32 sum (measured: the FMA kernels then reach 6.3 - 7.3x its error), so it would not measure fp32 error."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            return fn(*a)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


_MODEL = {}


def _model(kind, seed):
    """One model at a time: the codec (encoder, quantizer, decoder) or the redecoder, with its state dicts in float64 and
    float32 on the GPU."""
    import facodec_b200 as fb
    from facodec_b200 import synth
    key = (kind, seed)
    if key not in _MODEL:
        _MODEL.clear()
        torch.cuda.empty_cache()
        if kind == "codec":
            m, sds, parts = fb.build_model(), state_dicts(seed), ("encoder", "quantizer", "decoder")
        else:
            m, sds, parts = fb.build_model(stage="redecoder"), synth.synth_redecoder_state_dicts(seed), ("encoder", "decoder")
        for k in parts:
            m[k].load_state_dict(sds[k])
            m[k].eval()
        m[parts[0]]._engine.sync_weights(torch.device("cuda:0"))     # creates the handle the taps register on
        sd = {k: {d: _sd_to(sds[k], dt, "cuda") for d, dt in (("64", torch.float64), ("32", torch.float32))}
              for k in (("encoder", "decoder") if kind == "codec" else ("decoder",))}
        _MODEL[key] = (m, sd)
    return _MODEL[key]


# name -> (wseed, B, T, wave seed, golden fixture or None); the decoder input is the fixture's quantizer output "outs",
# or the quantizer output of the same call
CODEC_CASES = {n: (GOLDEN_CASES[n]["wseed"], GOLDEN_CASES[n]["B"], GOLDEN_CASES[n]["T"], GOLDEN_CASES[n]["xseed"], n)
               for n in ("b2_t7200", "b1_t96000", "b1_t7000_ragged", "b3_t1500_short")}
CODEC_CASES["b35_t2400"] = (1, 35, 2400, 35, None)          # 35 LSTM sequences: more than 32 per launch
CASE_ORDER = sorted(CODEC_CASES, key=lambda n: CODEC_CASES[n][0])


def _wave(case):
    from facodec_b200 import synth
    _, B, T, xseed, _ = CODEC_CASES[case]
    return synth.synth_waves(B, T, seed=xseed).cuda()


def _run_tapped(eng, names_shapes, fn, opts):
    """fn() under the route's options with a NaN-filled tap buffer [B][T][C] per (name, shape); returns (out, taps)."""
    taps = {n: torch.full(s, float("nan"), device="cuda") for n, s in names_shapes}
    out = _with_options(eng, opts, lambda: _tapped(eng, taps, fn))
    return out, taps


def _encoder_taps(B, T):
    shapes, t, ch = [("enc_conv0", (B, T, 64))], T, 64
    for i, s in enumerate(ENC_RATES):
        shapes += [(f"enc_block{i + 1}.res{j}", (B, t, ch)) for j in range(3)]
        t, ch = -(-t // s), 2 * ch
        shapes.append((f"enc_block{i + 1}", (B, t, ch)))
    return shapes + [("enc_lstm", (B, t, 1024))]


def _decoder_taps(B, Tf, with_lstm=True):
    shapes, t, ch = [("dec_conv0", (B, Tf, 1536))], Tf, 1536
    if with_lstm:
        shapes.append(("dec_lstm", (B, Tf, 1536)))
    for i, s in enumerate(DEC_RATES):
        t, ch = t * s, ch // 2
        shapes += [(f"dec_block{i + 1}.up", (B, t, ch))] + [(f"dec_block{i + 1}.res{j}", (B, t, ch)) for j in range(3)]
    return shapes


def _stats(y, y64, ref):
    return (y - y64).abs().max().item(), (ref - y64).abs().max().item(), y64.abs().max().item()


def check_steps(tag, steps, sd, x0, outs, bar, sep):
    """Teacher-forced: step k runs on outs of step k - 1 (x0 for the first) and is held to its bar.  outs: tap name ->
    GPU output [B][C][T] (fp32).  bar(name, kind) -> (class or "32", factor) of the max bar; sep(name, kind) -> (class,
    factor) of the separation bar or (None, None).  Returns the failed checks as (step, what, message)."""
    fails = []
    x = x0
    for name, kind, fn in steps:
        y = outs[name]
        if not torch.isfinite(y).all():
            fails.append((name, "finite", f"{tag} {name}: non-finite output"))
            break
        xin = x.double()
        with torch.no_grad():
            y64 = fn(sd["64"], xin, CLASSES[None])
            ref_kind, factor = bar(name, kind)
            ref = _fp32(fn, sd["32"], x.float(), CLASSES[None]).double() if ref_kind == "32" else \
                fn(sd["64"], xin, CLASSES[ref_kind])
            sep_cls, sep_f = sep(name, kind)
            ysep = fn(sd["64"], xin, CLASSES[sep_cls]) if sep_cls else None
        yd = y.double()
        err, eref, scale = _stats(yd, y64, ref)
        b = factor * eref + C * scale
        msg = f"STEP {tag} {name}: max|y-y64| {err:.3e}  max|y_{ref_kind}-y64| {eref:.3e}  err/ref {err / max(eref, 1e-300):.2f}" \
              f"  err/bar {err / b:.3f}"
        if ysep is not None:
            rk, rs = _rms(yd - y64), _rms(ysep - y64)
            msg += f"  rms/rms_{sep_cls} {rk / rs:.4f}"
        print(msg + f"  scale {scale:.3g}")
        if not err <= b:
            fails.append((name, "max", f"{tag} {name}: max|y - y64| = {err:.3e} > {b:.3e} ({factor} x {eref:.3e} "
                                       f"({ref_kind}) + floor)"))
        if ysep is not None and not rk <= sep_f * rs:
            fails.append((name, "sep", f"{tag} {name}: rms(y - y64) = {rk:.3e} > {sep_f} x {rs:.3e} ({sep_cls} class)"))
        x = y
    return fails


def _assert_no_fails(fails):
    for _, _, msg in fails:
        print("FAIL", msg)
    assert not fails, "; ".join(f[2] for f in fails)


def run_encoder(m, x, opts):
    eng = m.encoder._engine
    B, _, T = x.shape
    z, taps = _run_tapped(eng, _encoder_taps(B, T), lambda: m.encoder(x), opts)
    return z, taps


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(ENC_ROUTES))
@pytest.mark.parametrize("case", CASE_ORDER)
def test_encoder_steps_vs_fp64(case, route, built_lib):
    m, sd = _model("codec", CODEC_CASES[case][0])
    x = _wave(case)
    opts, factor = ENC_ROUTES[route]
    z, taps = run_encoder(m, x, opts)
    outs = {n: t.transpose(1, 2) for n, t in taps.items()}
    outs["z"] = z
    tag = f"enc {route} {case}"
    _assert_no_fails(check_steps(tag, encoder_steps(), sd["encoder"], x, outs, bar=lambda name, kind: ("32", factor),
                                      sep=lambda name, kind: ("bf16x3", SEP_ENC)))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASE_ORDER)
def test_encoder_tensor_cores1_equals_fma(case, built_lib):
    """tensor_cores = 1 runs no tensor-core kernel upstream of the VQ: every encoder tap and z bit-identical to
    tensor_cores = 0."""
    m, _ = _model("codec", CODEC_CASES[case][0])
    x = _wave(case)
    z1, t1 = run_encoder(m, x, {"tensor_cores": 1})
    z0, t0 = run_encoder(m, x, {"tensor_cores": 0})
    for n in t1:
        assert torch.equal(t1[n], t0[n]), f"{n}: tensor_cores = 1 differs from tensor_cores = 0"
    assert torch.equal(z1, z0)


_DEC_IN = {}


def _decoder_input(case, m):
    """[B][1024][Tf]: the fixture's "outs", or the quantizer output of the same encode."""
    if case not in _DEC_IN:
        _DEC_IN.clear()
        g = CODEC_CASES[case][4]
        if g is not None:
            _DEC_IN[case] = torch.from_numpy(load_golden(g)["outs"]).cuda()
        else:
            x = _wave(case)
            with torch.no_grad():
                _DEC_IN[case] = m.quantizer(m.encoder(x), x, n_c=2)[0].contiguous()
            torch.cuda.synchronize()
    return _DEC_IN[case]


PROMOTED = ("dec_conv0", "dec_block1.up")        # the decoder layers packed for the promoted kernel


def _dec_bar(route):
    _, conv_bar, unit_bar, _, _ = DEC_ROUTES[route]

    def bar(name, kind):
        if kind == "out" or (name in PROMOTED and route != "tensor_cores0"):
            return "32", F32                # the fp32 FMA kernel; the promoted fp16 hi + scaled-lo class
        b = unit_bar if kind == "unit" else conv_bar
        return ("32", b) if not isinstance(b, str) else (b, F_CLS)
    return bar


def _dec_sep(route):
    unit_sep = DEC_ROUTES[route][4]
    return lambda name, kind: ("fp16", SEP) if kind in ("conv0", "up") or (kind == "unit" and unit_sep) else (None, None)


def check_decoder(tag, steps, sd, z, y, taps, route):
    lstm_cfg = DEC_ROUTES[route][3]
    outs = {n: t.transpose(1, 2) for n, t in taps.items()}
    outs["y"] = y
    i = [s[0] for s in steps].index("dec_lstm") if "dec_lstm" in outs else None
    if i is not None:
        # the SLSTM step against test_gpu_lstm's bar of its class, on the dec_conv0 tap; the conv steps around it
        x = taps["dec_conv0"]
        ws = [sd["64"][f"model.1.lstm.{n}_l{l}"] for l in range(2) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]

        def ref(kind):
            if kind == "32":
                return _fp32(slstm_ref, x, ws, torch.float32)
            with torch.no_grad():
                return slstm_ref(x, ws) if kind == "64" else slstm_ref(x, ws, ih=kind[0], rec=kind[1])
        fails = check_steps(tag, steps[:i], sd, z, outs, _dec_bar(route), _dec_sep(route))
        fails += check_steps(tag, steps[i + 1:], sd, outs["dec_lstm"], outs, _dec_bar(route), _dec_sep(route))
        try:
            check_against_reference(taps["dec_lstm"], lstm_cfg, 1536, "tapped", f"{tag} dec_lstm", ref=ref)
        except AssertionError as e:
            fails.append(("dec_lstm", "lstm", str(e)))
    else:
        fails = check_steps(tag, steps, sd, z, outs, _dec_bar(route), _dec_sep(route))
    _assert_no_fails(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(DEC_ROUTES))
@pytest.mark.parametrize("case", CASE_ORDER)
def test_decoder_steps_vs_fp64(case, route, built_lib):
    m, sd = _model("codec", CODEC_CASES[case][0])
    z = _decoder_input(case, m)
    B, _, Tf = z.shape
    y, taps = _run_tapped(m.decoder._engine, _decoder_taps(B, Tf), lambda: m.decoder(z), DEC_ROUTES[route][0])
    check_decoder(f"dec {route} {case}", decoder_steps(), sd["decoder"], z, y, taps, route)


@pytest.mark.gpu
@pytest.mark.parametrize("route", REDEC_ROUTES)
@pytest.mark.parametrize("B,Tf", [(2, 24), (3, 5), (1, 320)])
def test_redecoder_decoder_steps_vs_fp64(B, Tf, route, built_lib):
    """The redecoder's non-causal decoder through fac_redecoder_decode, on the z of its own Redecoder."""
    m, sd = _model("redecoder", 0)
    cp, cc, tv = redecoder_inputs(B, Tf, 77 * B + Tf)
    with torch.no_grad():
        z = m.encoder(cp.cuda(), cc.cuda(), tv.cuda())
    y, taps = _run_tapped(m.decoder._engine, _decoder_taps(B, Tf, False), lambda: m.decoder(z), DEC_ROUTES[route][0])
    check_decoder(f"redec {route} B={B} Tf={Tf}", decoder_steps(False, False), sd["decoder"], z, y, taps, route)
