"""The two WaveNet stacks against a plain float64 restatement, on every precision route.

* The prosody branch (prosody_forward): mel[:, :20] -> melspec_linear -> WN (8 causal k = 5 layers, hidden 256) ->
  melspec_linear2 = f0, the input of the prosody VQ.  Its input is the "mel80" tap and its output the "f0_input" tap of
  the same FAquantizer call, so the mel front-end (held to fp64 by test_gpu_quantizer_kernels.py) is not in the error.
* The redecoder encoder (redecoder_forward): code embeddings -> cond_layer(timbre) (the B timbres are B rows of one GEMM)
  -> 16 non-causal k = 5 WN layers, each gate reading its own utterance's slice of g -> conv_out = z.

Kernels reached only through these stacks: wn_gate_kernel, wn_update_kernel, embed_sum_kernel.

References (all in this file).  The restatement runs each SConv1d as one product of unfolded input rows and the folded
weight, with the operands rounded as one precision class sees them (test_gpu_lstm._mm): exact, "bf16x3" (bf16 hi = rn(v),
lo = rn(v - hi), products hh + hl + lh) or "fp16" (one pass over fp16-rounded operands).  In exact mode it equals the
oracle's O.wavenet prosody branch and O.redecoder_forward in float64 (the *_reference_matches_the_oracle tests).
The GPU tests evaluate it on the GPU (cuBLAS float64, and float32 with TF32 off): y64 is float64 exact, y32 the same
stack in float32, y_bf16x3 / y_fp16 float64 with the class's operand rounding.  In the prosody branch the rounding
applies to the WN convs and melspec_linear2 (melspec_linear always runs the fp32 FMA kernel, its input rows being 80 floats apart); in the
redecoder the bf16x3 class rounds every conv and the fp16 class rounds the k = 5 in_layers to one fp16 pass and the rest
as bf16x3 (the one-pass blob the decoder's k = 7 convs take).

A worst-case bound is no use here: |W| propagated through the branch gives per-layer gains of about 22 (in_layers, l1
row sums) x 10 (res_skip), about 1e12 x the output scale over 8 layers.  So the bars, as in test_gpu_lstm.py, scale with
the run's own fp32 error or with an emulated rounding reference:

* fp32-grade routes:  max|y - y64| <= F max|y32 - y64| + C max|y64|, with F by arithmetic:
    F32 = 6 for the fp32 FMA kernels (tensor_cores = 0, and tensor_cores = 1 upstream of the VQ) and the promoted fp16
      hi + 2^11-scaled lo class (the prosody branch's default and encoder_tt = 1 routes);
    F_TF32X3 = 12 for the promoted 3xTF32 class (encoder_f16x2 = 0): its tf32 hi/lo split keeps fewer bits than the fp16
      pair and measures up to 9x the fp32 error where few frames make that error small;
    F_TF32X3_TRUNC = 160 for the non-promoted 3xTF32 class the redecoder runs with decoder_bf16 = 0: its tensor-core
      accumulation truncates (test_gpu_lstm.py uses 160 for the same class).  On this stack that route is no more
      accurate than the default bf16 hi/lo one (see below).
  F32 stays under the bf16x3/fp32 gap in max (7-15x on the CPU for the three regimes).
* Prosody class separation, every route:  rms(f0 - f64) <= 1/2 rms(f_bf16x3 - f64).
* Redecoder default route (bf16 hi/lo):  max|z - z64| <= F_BF16 max|z_bf16x3 - z64| + C max|z64|, F_BF16 = 2.5.
  No rms ratio against the bf16x3 model itself: like the LSTM's, it leaves out fp32 effects of its own size.
* Redecoder, every route:  rms(z - z64) <= 1/8 rms(z_fp16 - z64), which fails if a k = 5 conv runs the one-pass fp16
  class.
* Prosody codes: the fp64 f0 goes through test_gpu_quantizer_kernels._Chain with eps_in = the route's f0 bar; every frame
  whose prosody decision is decidable must get the fp64 code, and at least MIN_DECIDABLE of the frames must be decidable.
* tensor_cores = 1 keeps every layer upstream of the VQ on the FMA kernels, so its mel and f0 equal those of
  tensor_cores = 0 bit for bit.  This is what a prosody branch run without vq_critical breaks: its convs' precision class
  comes from their promoted packing, so on the default route that flag changes nothing, but with tensor_cores = 1 it moves
  the branch onto the tensor cores.

test_bars_separate_the_classes fixes, on the CPU for the seeds and shapes used, that these bars can tell the classes
apart: the bf16x3 prosody error is above the F32 bar in max and 14x the fp32 error in rms, and the fp16 redecoder error
38-56x the bf16x3 one in rms.

Regimes: the synthetic weights as they are, then in_layers weight_g x 8 (saturated gates; cond_layer x 8 as well in the
redecoder) and x 1/8 (nearly linear gates).  References run on the GPU (cuBLAS float64, and float32 with TF32 off).

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), ranges over every case:
  prosody branch     max|f0 - f64| / max|f32 - f64|    rms(f0 - f64) / rms(f_bf16x3 - f64)
    default            0.91 - 3.88                       0.090 - 0.153
    encoder_tt = 1     0.88 - 3.38                       0.090 - 0.153
    encoder_f16x2 = 0  1.86 - 9.13                       0.142 - 0.291
    tensor_cores 1, 0  1.08 - 2.60                       0.085 - 0.095
  Largest err / bar: 0.74 (encoder_f16x2 = 0), 0.61 on the other routes.  x8: 41 % of the gate pre-activations beyond
  |5|; as is and x 1/8: none.  Decidable prosody frames: 69 % or more of each case under its route's bar.
  redecoder z        max|z - z64| / max|z_ref - z64|   rms(z - z64) / rms(z_fp16 - z64)
    default            0.99 - 1.65 (z_ref = bf16x3)      0.025 - 0.068
    decoder_bf16 = 0   24 - 72 (z_ref = fp32)            0.028 - 0.071
    tensor_cores = 0   1.55 - 4.29 (z_ref = fp32)        0.002 - 0.004
  Largest err / bar: 0.70.  x8: 48 - 63 % of the gate pre-activations beyond |5|.
  The file's GPU tests took 43 s.
"""
import ctypes
import os

import pytest
import torch

from test_gpu_lstm import _mm
from test_gpu_quantizer_kernels import _Chain, _quantizer_vqs

# factors on the run's own fp32 error, per arithmetic (module docstring)
F32 = 6.0           # fp32 FMA kernels; the promoted fp16 hi + 2^11-scaled lo class
F_TF32X3 = 12.0     # the promoted 3xTF32 class (encoder_f16x2 = 0)
F_TF32X3_TRUNC = 160.0   # the non-promoted 3xTF32 class (decoder_bf16 = 0 downstream of the VQ)
F_BF16 = 2.5        # factor on the emulated bf16x3 error (redecoder default route)
C = 1e-7            # floor, relative to max|y64|
MIN_DECIDABLE = 0.4

HOP = 300
OPTION_DEFAULTS = {"tensor_cores": 2, "encoder_f16x2": 1, "encoder_tt": 0, "decoder_bf16": 1}
# route -> (options, factor of the fp32 bar; None = the redecoder's bf16x3 bar)
PROSODY_ROUTES = {"default": ({}, F32), "encoder_tt1": ({"encoder_tt": 1}, F32),
                  "encoder_f16x2_0": ({"encoder_f16x2": 0}, F_TF32X3), "tensor_cores1": ({"tensor_cores": 1}, F32),
                  "tensor_cores0": ({"tensor_cores": 0}, F32)}
REDEC_ROUTES = {"default": ({}, None), "decoder_bf16_0": ({"decoder_bf16": 0}, F_TF32X3_TRUNC),
                "tensor_cores0": ({"tensor_cores": 0}, F32)}
REGIMES = {"as_is": 1.0, "x8": 8.0, "x1_8": 0.125}
PROSODY_SEED, REDEC_SEED = 1, 0


def _threads():
    torch.set_num_threads(max(1, min(16, len(os.sched_getaffinity(0)))))


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _rms(d):
    return d.pow(2).mean().sqrt().item()


# ---------------------------------------------------------------------------------------------------------------------
# float64 restatement with per-conv operand rounding
# ---------------------------------------------------------------------------------------------------------------------
def _sconv(x, wb, mode=None, causal=True):
    """Stride-1 SConv1d (encodec.py:212-228, reflect padding through O._pad1d_reflect) on x [B][Cin][T] as one product of
    unfolded rows [B*T][Cin*K] and the folded weight [Cout][Cin*K]; `mode` rounds both operands (test_gpu_lstm._mm)."""
    from oracle import facodec_oracle as O
    w, b = wb
    B, Cin, T = x.shape
    K = w.shape[-1]
    if K > 1:
        pl = K - 1 if causal else (K - 1) - (K - 1) // 2
        x = O._pad1d_reflect(x, pl, K - 1 - pl)
    cols = x.unfold(2, K, 1).permute(0, 2, 1, 3).reshape(B * T, Cin * K)
    y = _mm(cols, w.reshape(w.shape[0], -1).t(), mode) + b
    return y.reshape(B, T, -1).transpose(1, 2)


def _wavenet(x, W, hidden, causal, mode, g=None, stats=None):
    """WN.forward (modules/wavenet.py:138-166, x_mask = 1, eval) on x [B][hidden][T]; g [B][2 hidden layers] is the
    cond_layer output (or None).  stats, if a list, receives (gate pre-activations beyond |5|, all of them)."""
    out = torch.zeros_like(x)
    n = len(W["in"])
    for i in range(n):
        pre = _sconv(x, W["in"][i], mode["in"], causal)
        if g is not None:
            pre = pre + g[:, i * 2 * hidden:(i + 1) * 2 * hidden, None]
        if stats is not None:
            stats.append(((pre.abs() > 5).sum().item(), pre.numel()))
        acts = torch.tanh(pre[:, :hidden]) * torch.sigmoid(pre[:, hidden:])
        rs = _sconv(acts, W["rs"][i], mode["rs"], causal)
        if i < n - 1:
            x = x + rs[:, :hidden]
            out = out + rs[:, hidden:]
        else:
            out = out + rs
    return out


def _sd_to(sd, dtype, device):
    return {k: (v.to(device, dtype) if v.is_floating_point() else v.to(device)) for k, v in sd.items()}


def prosody_weights(sd, dtype=torch.float64, device="cpu"):
    from oracle import facodec_oracle as O
    s = _sd_to(sd, dtype, device)
    W = lambda p: (O._wn_weight(s, p), s[p + ".bias"])
    return {"lin": W("melspec_linear.conv.conv"), "lin2": W("melspec_linear2.conv.conv"),
            "in": [W(f"melspec_encoder.in_layers.{i}.conv.conv") for i in range(8)],
            "rs": [W(f"melspec_encoder.res_skip_layers.{i}.conv.conv") for i in range(8)]}


def redecoder_weights(sd, dtype=torch.float64, device="cpu"):
    from oracle import facodec_oracle as O
    s = _sd_to(sd, dtype, device)
    W = lambda p: (O._wn_weight(s, p), s[p + ".bias"])
    return {"cond": W("encoder.cond_layer.conv.conv"), "out": W("conv_out"),
            "in": [W(f"encoder.in_layers.{i}.conv.conv") for i in range(16)],
            "rs": [W(f"encoder.res_skip_layers.{i}.conv.conv") for i in range(16)],
            "emb_p": s["prosody_embed.0.weight"], "emb_c": [s[f"content_embed.{i}.weight"] for i in range(2)]}


# operand rounding per conv family of each precision class
PROSODY_CLASS = {None: {"lin": None, "in": None, "rs": None, "lin2": None},
                 "bf16x3": {"lin": None, "in": "bf16x3", "rs": "bf16x3", "lin2": "bf16x3"}}
REDEC_CLASS = {None: {"cond": None, "in": None, "rs": None, "out": None},
               "bf16x3": {"cond": "bf16x3", "in": "bf16x3", "rs": "bf16x3", "out": "bf16x3"},
               "fp16": {"cond": "bf16x3", "in": "fp16", "rs": "bf16x3", "out": "bf16x3"}}


def prosody_ref(W, mel, cls=None, stats=None):
    """The prosody branch on mel [B][Tm][80] (the mel80 tap) in mel's dtype -> f0 [B][Tm][1024]."""
    m = PROSODY_CLASS[cls]
    x = _sconv(mel[..., :20].transpose(1, 2), W["lin"], m["lin"])
    x = _wavenet(x, W, 256, True, m, stats=stats)
    return _sconv(x, W["lin2"], m["lin2"]).transpose(1, 2)


def redecoder_ref(W, cp, cc, tv, use_p, use_c, n_c, cls=None, stats=None):
    """Redecoder.forward (modules/redecoder.py:35-48) on codes cp [B][1][T], cc [B][>= n_c][T] and timbre tv [B][1024]
    in tv's dtype -> z [B][1024][T]."""
    m = REDEC_CLASS[cls]
    B, _, T = cp.shape
    pe = torch.zeros(B, T, 512, dtype=tv.dtype, device=tv.device)
    ce = torch.zeros_like(pe)
    if use_p:
        pe = pe + W["emb_p"][cp[:, 0]]
    if use_c:
        for i in range(n_c):
            ce = ce + W["emb_c"][i][cc[:, i]]
    x = (pe + ce).transpose(1, 2)
    g = _sconv(tv[:, :, None], W["cond"], m["cond"])[:, :, 0]
    x = _wavenet(x, W, 512, False, m, g=g, stats=stats)
    return _sconv(x, W["out"], m["out"])


# ---------------------------------------------------------------------------------------------------------------------
# weights, regimes, inputs
# ---------------------------------------------------------------------------------------------------------------------
def prosody_sd(regime):
    from conftest import state_dicts
    sd = dict(state_dicts(PROSODY_SEED)["quantizer"])
    for i in range(8):
        k = f"melspec_encoder.in_layers.{i}.conv.conv.weight_g"
        sd[k] = sd[k] * REGIMES[regime]
    return sd


_RED_SDS = {}


def redecoder_sds(regime):
    from facodec_b200 import synth
    if not _RED_SDS:
        _RED_SDS["base"] = synth.synth_redecoder_state_dicts(REDEC_SEED)
    sds = dict(_RED_SDS["base"])
    enc = dict(sds["encoder"])
    keys = [f"encoder.in_layers.{i}.conv.conv.weight_g" for i in range(16)] + ["encoder.cond_layer.conv.conv.weight_g"]
    for k in keys:
        enc[k] = enc[k] * REGIMES[regime]
    sds["encoder"] = enc
    return sds


def redecoder_inputs(B, T, seed):
    """Codes with 0 and 1023 in every table (when B T >= 2) and a distinct N(0, 1) timbre per utterance."""
    g = torch.Generator().manual_seed(seed)
    cp = torch.randint(0, 1024, (B, 1, T), generator=g)
    cc = torch.randint(0, 1024, (B, 2, T), generator=g)
    for t in (cp, cc):
        t[0, :, 0] = 0
        t[-1, :, -1] = 1023
    tv = torch.randn(B, 1024, generator=g)
    return cp, cc, tv


def _cpu_mel(B, T, seed):
    from facodec_b200 import synth
    from conftest import state_dicts
    from oracle import facodec_oracle as O
    x = synth.synth_waves(B, T, seed=seed)
    sd = _sd_to(state_dicts(PROSODY_SEED)["quantizer"], torch.float64, "cpu")
    return O.mel_preprocess(sd, x.double(), n_bins=80).transpose(1, 2).contiguous()      # [B][Tm][80]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatement against the oracle, and the separations the GPU bars rely on
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Tm", [3, 24])
def test_prosody_reference_matches_the_oracle(Tm):
    """Tm = 3 takes pad1d's short-input branch at k = 5 causal."""
    from oracle import facodec_oracle as O
    _threads()
    mel = _cpu_mel(2, max(1025, Tm * HOP + 7), 5)
    sd = _sd_to(prosody_sd("as_is"), torch.float64, "cpu")
    with torch.no_grad():
        f = O.sconv1d(mel[..., :20].transpose(1, 2), sd, "melspec_linear.conv.conv")
        f = O.wavenet(sd, f)
        ref = O.sconv1d(f, sd, "melspec_linear2.conv.conv").transpose(1, 2)
    got = prosody_ref(prosody_weights(prosody_sd("as_is")), mel)
    assert (got - ref).abs().max().item() <= 1e-14 * ref.abs().max().item()


@pytest.mark.parametrize("use_p,use_c,n_c,T", [(1, 1, 2, 2), (0, 1, 1, 20), (1, 0, 2, 5)])
def test_redecoder_reference_matches_the_oracle(use_p, use_c, n_c, T):
    """T = 2 takes the short-input branch of the non-causal 2 / 2 reflect pad."""
    from oracle import facodec_oracle as O
    _threads()
    sd = redecoder_sds("as_is")["encoder"]
    cp, cc, tv = redecoder_inputs(2, T, 11 + T)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)          # the oracle's embedding sums start from default-dtype zeros
    try:
        with torch.no_grad():
            ref = O.redecoder_forward(_sd_to(sd, torch.float64, "cpu"), cp, cc, tv.double(), use_p_code=bool(use_p),
                                      use_c_code=bool(use_c), n_c=n_c)
    finally:
        torch.set_default_dtype(prev)
    got = redecoder_ref(redecoder_weights(sd), cp, cc, tv.double(), use_p, use_c, n_c)
    assert (got - ref).abs().max().item() <= 1e-14 * ref.abs().max().item()


def _f0_bar(err32, scale, factor=F32):
    return factor * err32 + C * scale


@pytest.mark.parametrize("regime", list(REGIMES))
def test_bars_separate_the_classes(regime):
    """For the seeds, regimes and the shapes used: the prosody branch's bf16x3 error is far above the F32 bar (max) and
    above twice the fp32 error (rms), the redecoder's fp16 error far above its bf16x3 error (rms), and enough prosody
    decisions stay decidable with eps_in = the loosest f0 bar (F_TF32X3) for the code check to mean something."""
    from conftest import state_dicts
    _threads()
    mel = _cpu_mel(3, 24 * HOP + 123, 17)
    sd = prosody_sd(regime)
    W64, W32 = prosody_weights(sd), prosody_weights(sd, torch.float32)
    with torch.no_grad():
        f64 = prosody_ref(W64, mel)
        f32 = prosody_ref(W32, mel.float()).double()
        fb = prosody_ref(W64, mel, "bf16x3")
    scale = f64.abs().max().item()
    e32, eb = (f32 - f64).abs().max().item(), (fb - f64).abs().max().item()
    r32, rb = _rms(f32 - f64), _rms(fb - f64)
    bar = _f0_bar(e32, scale)
    p = _Chain(_quantizer_vqs(state_dicts(PROSODY_SEED)["quantizer"])[0:1], f64.reshape(-1, 1024),
               eps_in=torch.full((f64.shape[0] * f64.shape[1], 1024), _f0_bar(e32, scale, F_TF32X3),
                                 dtype=torch.float64))
    frac = p.decidable().double().mean().item()
    print(f"SEP prosody {regime}: max f32 {e32:.3e} bf16x3 {eb:.3e} (x{eb / bar:.1f} the bar)  rms f32 {r32:.3e} "
          f"bf16x3 {rb:.3e} (x{rb / r32:.1f})  scale {scale:.3f}  decidable {frac:.3f}")
    assert eb >= 1.15 * bar and rb >= 8 * r32
    assert frac >= MIN_DECIDABLE + 0.1                # with the loosest f0 bar
    if regime == "x1_8":
        return                                           # the redecoder runs as_is and x8 only
    sds = redecoder_sds(regime)["encoder"]
    W64 = redecoder_weights(sds)
    W32 = redecoder_weights(sds, torch.float32)
    cp, cc, tv = redecoder_inputs(2, 60, 3)
    with torch.no_grad():
        z64 = redecoder_ref(W64, cp, cc, tv.double(), 1, 1, 2)
        z32 = redecoder_ref(W32, cp, cc, tv, 1, 1, 2).double()
        zb = redecoder_ref(W64, cp, cc, tv.double(), 1, 1, 2, "bf16x3")
        zh = redecoder_ref(W64, cp, cc, tv.double(), 1, 1, 2, "fp16")
    scale = z64.abs().max().item()
    e32, eb = (z32 - z64).abs().max().item(), (zb - z64).abs().max().item()
    r32, rb, rh = _rms(z32 - z64), _rms(zb - z64), _rms(zh - z64)
    print(f"SEP redecoder {regime}: max f32 {e32:.3e} bf16x3 {eb:.3e}  rms f32 {r32:.3e} bf16x3 {rb:.3e} fp16 {rh:.3e} "
          f"(x{rh / rb:.1f})  scale {scale:.3f}")
    assert eb >= 1.15 * _f0_bar(e32, scale)       # the F32 bar of the fp32-grade routes excludes the bf16x3 class
    assert rh >= 16 * rb                           # the 1/8 fp16 bar leaves twice the bf16x3 class's rms


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _with_options(eng, opts, fn, defaults=None):
    """fn() with the engine options opts set, each restored to its value in defaults (OPTION_DEFAULTS) afterwards."""
    defaults = OPTION_DEFAULTS if defaults is None else defaults
    try:
        for k, v in opts.items():
            eng.set_option(k, v)
        return fn()
    finally:
        for k in opts:
            eng.set_option(k, defaults[k])


_CODEC = {}


def _codec(regime):
    """One codec model for the module, its quantizer reloaded with the regime's weights when the regime changes."""
    import facodec_b200 as fb
    from conftest import state_dicts
    if "m" not in _CODEC:
        m = fb.build_model()
        sds = state_dicts(PROSODY_SEED)
        for k in ("encoder", "decoder"):
            m[k].load_state_dict(sds[k])
            m[k].eval()
        _CODEC["m"] = m
    m = _CODEC["m"]
    if _CODEC.get("regime") != regime:
        m.quantizer.load_state_dict(prosody_sd(regime))
        m.quantizer.eval()
        m.quantizer._engine.sync_weights(torch.device("cuda:0"))
        _CODEC["regime"] = regime
        _CODEC["W"] = {k: prosody_weights(prosody_sd(regime), d, "cuda") for k, d in (("64", torch.float64),
                                                                                  ("32", torch.float32))}
    return m, _CODEC["W"]


def _tapped(eng, taps, fn):
    """Runs fn with the named debug taps copying into the given tensors; synchronises."""
    try:
        for name, t in taps.items():
            eng.L.fac_debug_tap(eng.handle, name.encode(), _p(t), t.numel())
        out = fn()
        torch.cuda.synchronize()
        return out
    finally:
        for name in taps:
            eng.L.fac_debug_tap(eng.handle, name.encode(), None, 0)


def _run_quantizer(m, x, z, opts):
    eng = m.quantizer._engine
    B, Tm = x.shape[0], x.shape[-1] // HOP
    mel = torch.full((B, Tm, 80), float("nan"), device="cuda")
    f0 = torch.full((B, Tm, 1024), float("nan"), device="cuda")
    out = _with_options(eng, opts, lambda: _tapped(eng, {"mel80": mel, "f0_input": f0},
                                                   lambda: m.quantizer(z, x, n_c=1, return_codes=True)))
    return mel, f0, out[5][0]


def _fp32_ref(fn, *a):
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return fn(*a)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32


def check_f0(tag, W, f0, mel, factor=F32, stats=None):
    """Holds f0 [B][Tm][1024] (GPU) to the fp32 bar and the class-separation bar; returns (f64, bar)."""
    assert torch.isfinite(f0).all(), f"{tag}: non-finite f0"
    with torch.no_grad():
        f64 = prosody_ref(W["64"], mel.double(), stats=stats)
        f32 = _fp32_ref(prosody_ref, W["32"], mel.float()).double()
        fb = prosody_ref(W["64"], mel.double(), "bf16x3")
    d = f0.double() - f64
    err, err32, scale = d.abs().max().item(), (f32 - f64).abs().max().item(), f64.abs().max().item()
    rk, rb = _rms(d), _rms(fb - f64)
    bar = _f0_bar(err32, scale, factor)
    sat = f"  |pre| > 5: {sum(s[0] for s in stats) / sum(s[1] for s in stats):.3f}" if stats else ""
    print(f"F0 {tag}: max|f0-f64| {err:.3e}  max|f32-f64| {err32:.3e}  err/err32 {err / max(err32, 1e-300):.2f}  "
          f"err/bar {err / bar:.3f}  rms(f0-f64)/rms(fb-f64) {rk / rb:.3f}  scale {scale:.3f}{sat}")
    assert err <= bar, f"{tag}: max|f0 - f64| = {err:.3e} > {bar:.3e}"
    assert rk <= 0.5 * rb, f"{tag}: rms(f0 - f64) = {rk:.3e} > 1/2 x {rb:.3e} (bf16x3 class)"
    return f64, bar


def check_prosody_codes(tag, f64, bar, codes_p, n_frames_min=1):
    """Frames [B][Tq] of codes_p whose prosody decision is decidable with eps_in = bar get the fp64 code."""
    from conftest import state_dicts
    B, Tq, _ = f64.shape
    frames = f64.reshape(B * Tq, 1024).cpu()
    p = _Chain(_quantizer_vqs(state_dicts(PROSODY_SEED)["quantizer"])[0:1], frames,
               eps_in=torch.full_like(frames, bar))
    ok = p.decidable()
    got = codes_p.reshape(B * Tq).cpu()
    n_ok = int(ok.sum())
    print(f"CODES {tag}: decidable {n_ok} of {B * Tq}")
    assert n_ok >= max(n_frames_min, int(MIN_DECIDABLE * B * Tq)), f"{tag}: {n_ok} of {B * Tq} decidable"
    assert torch.equal(got[ok], p.codes[0][ok]), f"{tag}: {int((got[ok] != p.codes[0][ok]).sum())} decidable codes differ"


# (regime, Tm, T): Tm <= 4 takes pad1d's short-input branch; the others are not multiples of 300 samples
PROSODY_SHAPES = [(3, 1025), (4, 1200), (5, 1500), (64, 64 * HOP + 299), (65, 65 * HOP + 1), (128, 128 * HOP + 150),
                  (129, 129 * HOP + 77)]
PROSODY_CASES = [("as_is", Tm, T) for Tm, T in PROSODY_SHAPES] + \
                [(r, Tm, T) for r in ("x8", "x1_8") for Tm, T in PROSODY_SHAPES if Tm in (4, 65)]


@pytest.mark.gpu
@pytest.mark.parametrize("regime,Tm,T", PROSODY_CASES)
def test_prosody_branch_vs_fp64(regime, Tm, T, built_lib):
    """Every route on the same waveform: f0 against fp64, the prosody codes on decidable frames, and tensor_cores = 1
    bit-identical to tensor_cores = 0 (both keep the branch on the FMA kernels)."""
    from facodec_b200 import synth
    m, W = _codec(regime)
    B = 3
    x = synth.synth_waves(B, T, seed=T + 31).cuda()
    z = torch.randn(B, 1024, Tm + 2, generator=torch.Generator().manual_seed(T)).cuda()
    fma = {}
    for route, (opts, factor) in PROSODY_ROUTES.items():
        mel, f0, cp = _run_quantizer(m, x, z, opts)
        tag = f"{route} {regime} B={B} Tm={Tm}"
        stats = [] if route == "default" else None
        f64, bar = check_f0(tag, W, f0, mel, factor, stats)
        check_prosody_codes(tag, f64, bar, cp)
        if route.startswith("tensor_cores"):
            fma[route] = (mel, f0, cp)
    (m1, f1, c1), (m0, f0_, c0) = fma["tensor_cores1"], fma["tensor_cores0"]
    assert torch.equal(m1, m0) and torch.equal(f1, f0_) and torch.equal(c1, c0), \
        "tensor_cores = 1 must run the prosody branch on the same FMA kernels as tensor_cores = 0"


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["default", "tensor_cores0"])
def test_prosody_branch_ragged_lanes(route, built_lib):
    """One Codec.forward(lengths=...) call: lane b's f0 rows t < Tm_b against fp64 on its own mel rows.  The lengths give
    Tm_b = 24, 3 (the short-input branch), 10 and 17."""
    from facodec_b200 import synth
    import facodec_b200 as fb
    m, W = _codec("as_is")
    eng = m.quantizer._engine
    lens = [7300, 1025, 3299, 5111]
    B, T = len(lens), max(lens)
    Tm = T // HOP
    x = synth.synth_waves(B, T, seed=404).cuda()
    mel = torch.full((B, Tm, 80), float("nan"), device="cuda")
    f0 = torch.full((B, Tm, 1024), float("nan"), device="cuda")
    codec = fb.Codec(m)
    opts, factor = PROSODY_ROUTES[route]
    _with_options(eng, opts,
                  lambda: _tapped(eng, {"mel80": mel, "f0_input": f0}, lambda: codec.forward(x, n_c=2, lengths=lens)))
    for b, n in enumerate(lens):
        tm = n // HOP
        check_f0(f"ragged {route} lane {b} Tm_b={tm}", W, f0[b:b + 1, :tm], mel[b:b + 1, :tm], factor)


REDEC_CODE_CASES = [(1, 1, 2), (0, 1, 1), (1, 1, 1), (1, 0, 2)]
REDEC_CASES = [("default", "as_is", u, 2, T) for u in REDEC_CODE_CASES for T in (1, 2, 3, 5, 64, 65, 200)] + \
              [("default", "as_is", (1, 1, 2), B, 3) for B in (1, 3, 64, 65, 128, 129)] + \
              [("default", "x8", u, B, T) for u in ((1, 1, 2), (0, 1, 1)) for B, T in ((2, 2), (3, 65))] + \
              [(r, g, (1, 1, 2), B, T) for r in ("decoder_bf16_0", "tensor_cores0") for g in ("as_is", "x8")
               for B, T in ((2, 2), (3, 65), (65, 3))] + \
              [(r, "as_is", (0, 1, 1), 3, 200) for r in ("decoder_bf16_0", "tensor_cores0")]
REDEC_CASES.sort(key=lambda c: c[1] != "as_is")


_RED = {}


def _redecoder(regime):
    import facodec_b200 as fb
    if "m" not in _RED:
        _RED["m"] = fb.build_model(stage="redecoder")
    m = _RED["m"]
    if _RED.get("regime") != regime:
        sds = redecoder_sds(regime)
        for k in ("encoder", "decoder"):
            m[k].load_state_dict(sds[k])
            m[k].eval()
        _RED["regime"] = regime
        _RED["W"] = {k: redecoder_weights(sds["encoder"], d, "cuda") for k, d in (("64", torch.float64),
                                                                              ("32", torch.float32))}
    return m, _RED["W"]


@pytest.mark.gpu
@pytest.mark.parametrize("route,regime,codes,B,T", REDEC_CASES)
def test_redecoder_vs_fp64(route, regime, codes, B, T, built_lib):
    """z of Redecoder.forward against the fp64 restatement; every utterance has its own timbre."""
    use_p, use_c, n_c = codes
    m, W = _redecoder(regime)
    cp, cc, tv = redecoder_inputs(B, T, 1000 * B + T)
    eng = m.encoder._engine
    opts, factor = REDEC_ROUTES[route]
    z = _with_options(eng, opts, lambda: m.encoder(cp.cuda(), cc.cuda(), tv.cuda(), use_p_code=bool(use_p),
                                                                    use_c_code=bool(use_c), n_c=n_c))
    torch.cuda.synchronize()
    assert torch.isfinite(z).all()
    cpd, ccd, tvd = cp.cuda(), cc.cuda(), tv.cuda().double()
    stats = []
    with torch.no_grad():
        z64 = redecoder_ref(W["64"], cpd, ccd, tvd, use_p, use_c, n_c, stats=stats)
    d = z.double() - z64
    err, scale = d.abs().max().item(), z64.abs().max().item()
    sat = sum(s[0] for s in stats) / sum(s[1] for s in stats)
    tag = f"{route} {regime} codes={codes} B={B} T={T}"
    with torch.no_grad():
        zh = redecoder_ref(W["64"], cpd, ccd, tvd, use_p, use_c, n_c, "fp16")
    rk, rh = _rms(d), _rms(zh - z64)
    if factor is None:
        with torch.no_grad():
            zb = redecoder_ref(W["64"], cpd, ccd, tvd, use_p, use_c, n_c, "bf16x3")
        errb = (zb - z64).abs().max().item()
        bar = F_BF16 * errb + C * scale
        what = f"max|zb-z64| {errb:.3e}  err/errb {err / errb:.2f}"
    else:
        z32 = _fp32_ref(redecoder_ref, W["32"], cpd, ccd, tv.cuda(), use_p, use_c, n_c).double()
        err32 = (z32 - z64).abs().max().item()
        bar = factor * err32 + C * scale
        what = f"max|z32-z64| {err32:.3e}  err/err32 {err / err32:.2f}"
    print(f"RED {tag}: max|z-z64| {err:.3e}  {what}  err/bar {err / bar:.3f}  rms(z-z64)/rms(zh-z64) {rk / rh:.4f}  "
          f"scale {scale:.2f}  |pre| > 5: {sat:.3f}")
    assert err <= bar, f"{tag}: max|z - z64| = {err:.3e} > {bar:.3e}"
    assert rk <= rh / 8, f"{tag}: rms(z - z64) = {rk:.3e} > 1/8 x {rh:.3e} (one-pass fp16 class)"
