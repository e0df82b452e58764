"""The predictor heads against a plain float64 restatement: alias-free SnakeBeta, the CNNLSTM trunks and their linears,
FApredictors at the training geometry.

Kernels and engine paths reached only through these heads: alias_free_act_kernel (fac_alias_free_act and every
Activation1d of a head), fac_head_forward (symmetric zero-padded dilated k = 7 convs, a linear over B*T frames as the rows
of one lane, launch_mean_pool without lane lengths, the engine's own fp64 -> fp32 Kaiser-sinc filter) and fac_add3.

References (all in this file).  The restatement runs Activation1d as UpSample1d(2, 12) (replicate pad 5, the 12-tap
Kaiser-sinc filter as a stride-2 transposed conv, x 2, crop 15 / 15), SnakeBeta x + 1 / (exp(beta) + 1e-9) sin^2(exp(alpha)
x), DownSample1d(2, 12) (replicate pad (5, 6), stride 2), written as gathers and tap sums so that no library conv (and no
TF32) is involved.  The filter is evaluated in float64.  A ResidualUnit is act -> k = 7 conv (dilation d, zero padding 3d)
-> act -> 1x1 conv -> + x; CNNLSTM is three of them (d = 1, 2, 3), the final act, the transpose, an optional mean over
T and the linear heads.  Each conv and linear is one product of unfolded rows and the folded weight (weight norm folded
in float64 from the fp32 weight_v / weight_g) through test_gpu_lstm._mm, so one flag rounds the operands as a precision
class sees them: exact, "bf16x3" (hi / lo split, hh + hl + lh) or "fp16" (one pass).  The rounding goes only to the
layers the product sends to the tensor cores, as fac_debug_tc_plan decides it (it refuses the Cout = 1 f0 / uv linears
and the Cout = 50 test linears, which run the fp32 FMA kernels): those stay exact in every class.  In exact mode the
restatement equals O.alias_free_act, O.cnnlstm_forward and O.fa_predictors_forward run in float64 (the *_matches_the_oracle
tests; the oracle's filter is then its float64 twin).  On the GPU y64 is the float64 restatement (cuBLAS), y32 the same in
float32 with TF32 off, y_bf16x3 / y_fp16 float64 with the class's operand rounding.

Bars (factors from test_gpu_wavenet.py):
* Activation1d, identity: elementwise |y - y64| <= 2 F1 S Xw ((g12 + u)(1 + 10u) + g6 (1 + u) + u), u = 2^-24,
  g_n = n u / (1 - n u), F1 = sum |f|, S = the larger of sum |f| over the even and over the odd taps, Xw = max |x| over
  the 13 input samples output t reaches: the 6 FMAs of an up-sampled sample, the 12 of an output, and the fp32 rounding
  of the taps, to first order.  It is an a-priori bound, not a fitted tolerance.
* Activation1d, SnakeBeta:  max|y - y64| <= F32 max|y32 - y64| + C max|y64|.
* Constant input comes back within 8 ulp of the constant at every sample: each parity's taps sum to 1/2, so the
  replicate padding at both ends keeps it exact up to rounding.
* Heads, default route (bf16 hi/lo):  max|y - y64| <= F_BF16 max|y_bf16x3 - y64| + C max|y64|;
  tensor_cores = 0 (fp32 FMA):  F32 x the fp32 error;  decoder_bf16 = 0 (non-promoted 3xTF32):  F_TF32X3_TRUNC x it.
  An output no tensor-core layer feeds (the 16 -> 1 and 64 -> 50 linears) takes the F32 bar on every route.
* Heads, every route:  rms(y - y64) <= 1/8 rms(y_fp16 - y64), which fails if any head layer runs the one-pass fp16
  class.
* in_dim 1024 takes wider factors: F_BF16_1024 = 16, F32_1024 = 12, F_TF32X3_TRUNC_1024 = 320 and an rms bar of 1/2.
  Each k = 7 output there is a chain of K = 7168 products (1792 at in_dim 256).  The non-promoted tensor-core classes
  accumulate without promotion in a truncating accumulator, which the operand-rounding model leaves out, and the fp32
  FMA kernel sums its chain in one serial order where cuBLAS blocks it; both errors grow with K.  Pooled outputs average
  the rounding errors of T frames but not the one-sided truncation, so their ratios are the largest.  Measured maxima:
  11.7 (default, the pooled 1024 -> 50 head), 8.0 (tensor_cores = 0), 204 (decoder_bf16 = 0, pooled) and an rms ratio
  of 0.28 (decoder_bf16 = 0, pooled); 4.3 on the f0 output of FApredictors at the training geometry.
test_bars_separate_the_classes fixes on the CPU, for the seeds and shapes used, that these bars tell the classes apart.

Exact properties: batch invariance (an utterance alone equals its rows of the batch, per-frame and pooled outputs),
repeatability, and no bit moved by tensor_cores 1 vs 2, decoder_conv7_fp16 0 vs 1 or tc_occ2_maxn 0 vs 128.  Outputs
written through views into NaN-guarded buffers leave the guards untouched; a workspace full of NaN from an earlier,
larger call changes no bit.  fac_add3 equals torch's fp32 (a + b) + c bit for bit.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), ranges over every case:
  Activation1d identity   max err / a-priori bound 0.04 - 0.16;  constant rows 1 - 2 ulp
  Activation1d SnakeBeta  max|y - y64| / max|y32 - y64|: synth 0.49 - 3.11, log alpha 2 0.67 - 0.99,
                          log beta -3 0.85 - 0.98, x8 0.80 - 1.41;  largest err / bar 0.37
  heads, in_dim <= 256    err / err_ref: default 0.61 - 2.44 (bf16x3), decoder_bf16 = 0 0.56 - 69 (fp32),
                          tensor_cores = 0 0.22 - 3.83 (fp32);  largest err / bar 0.81
  heads, in_dim 1024      default 1.13 - 11.7, decoder_bf16 = 0 49 - 204, tensor_cores = 0 1.59 - 8.02;
                          largest err / bar 0.73;  rms(y - y64) / rms(y_fp16 - y64) up to 0.14 (default), 0.28
  The file's GPU tests took 46 s.
Findings: none in the kernels.  Moving the k = 7 convs' pad_right changes nothing, since zero padding reads no row
outside [0, T) whatever the pads are.
"""
import ctypes
import functools
import math
import os

import pytest
import torch
import torch.nn.functional as F

from test_gpu_lstm import _mm
from test_gpu_wavenet import C, F32, F_BF16, F_TF32X3_TRUNC

FAC_ERR_INVALID, FAC_ERR_STATE, FAC_ERR_UNSUPPORTED = -1, -2, -4
OPTION_DEFAULTS = {"tensor_cores": 2, "decoder_bf16": 1, "decoder_conv7_fp16": 1, "tc_occ2_maxn": 0}
# route -> (options, factor on the fp32 error; None = the bf16x3 bar)
ROUTES = {"default": ({}, None), "decoder_bf16_0": ({"decoder_bf16": 0}, F_TF32X3_TRUNC),
          "tensor_cores0": ({"tensor_cores": 0}, F32)}
# in_dim 1024 (K = 7168 per k = 7 output, module docstring): wider factors of the default and FMA routes, and of the
# fp16 rms bar
F_BF16_1024, F32_1024, F_TF32X3_TRUNC_1024, RMS_FP16_1024 = 16.0, 12.0, 320.0, 0.5
U32 = 2.0 ** -24


def _threads():
    torch.set_num_threads(max(1, min(16, len(os.sched_getaffinity(0)))))


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _rms(d):
    return d.double().pow(2).mean().sqrt().item()


# ---------------------------------------------------------------------------------------------------------------------
# float64 restatement with per-layer operand rounding
# ---------------------------------------------------------------------------------------------------------------------
def aa_filter(dtype=torch.float64, device="cpu"):
    """kaiser_sinc_filter1d(cutoff 0.25, half_width 0.3, 12 taps) (alias_free_torch/filter.py:27-58) in float64."""
    half = 6
    A = 2.285 * (half - 1) * math.pi * (4 * 0.3) + 7.95
    beta = 0.1102 * (A - 8.7) if A > 50.0 else (0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0) if A >= 21.0 else 0.0)
    win = torch.kaiser_window(12, periodic=False, beta=beta, dtype=torch.float64)
    t = torch.arange(-half, half, dtype=torch.float64) + 0.5
    f = 2 * 0.25 * win * torch.sinc(2 * 0.25 * t)
    return (f / f.sum()).to(device, dtype)


def _clamped(x, lo, n, size):
    """x[..., clamp(lo + i, 0, size - 1)] for i < n: replicate padding as a gather."""
    idx = (torch.arange(n, device=x.device) + lo).clamp(0, size - 1)
    return x[..., idx]


def aa_act(x, f, la=None, lb=None):
    """Activation1d (alias_free_torch/act.py:24-29) on x [B][C][T] in x's dtype; la / lb are SnakeBeta's log-scale alpha
    / beta [C] (modules/quantize.py:78-88), or None for the identity."""
    T = x.shape[-1]
    xp = _clamped(x, -5, T + 10, T).unfold(-1, 6, 1)                  # [B][C][T + 5][6]: xp[j + q], xp = replicate pad 5
    # conv_transpose1d stride 2 then crop 15: u[2j] = 2 sum_l xp[j + 7 - l] f[2l + 1], u[2j + 1] = 2 sum_l xp[j + 8 - l] f[2l]
    ue = 2 * (xp[..., 2:2 + T, :] * f[1::2].flip(0)).sum(-1)
    uo = 2 * (xp[..., 3:3 + T, :] * f[0::2].flip(0)).sum(-1)
    u = torch.stack([ue, uo], -1).reshape(*x.shape[:-1], 2 * T)
    if la is not None:
        a, b = torch.exp(la)[:, None], torch.exp(lb)[:, None]
        u = u + (1.0 / (b + 1e-9)) * torch.sin(u * a).pow(2)
    d = _clamped(u, -5, 2 * T + 11, 2 * T)                             # replicate pad (5, 6)
    return (d.unfold(-1, 12, 2) * f).sum(-1)


@functools.lru_cache(maxsize=None)
def _tc_eligible(Cin, Cout, K, dil, Tout):
    """Whether the product sends this layer to the tensor cores (fac_debug_tc_plan, bf16 class)."""
    from facodec_b200 import _lib
    out = (ctypes.c_int * 8)()
    rc = _lib.load().fac_debug_tc_plan(Cin, Cout, K, dil, 1, Tout, 2, 0, out)
    assert rc in (0, FAC_ERR_UNSUPPORTED), rc
    return rc == 0


def _mode(cls, Cin, Cout, K, dil, Tout):
    return cls if cls is not None and _tc_eligible(Cin, Cout, K, dil, Tout) else None


def _conv(x, wb, dil, cls):
    """nn.Conv1d(C, C', K, dilation=dil, padding=(K - 1) dil // 2) (zeros; modules/quantize.py:90-104) on x [B][C][T] as
    one product of unfolded rows [B*T][C*K] and the folded weight."""
    w, b = wb
    B, Cin, T = x.shape
    Cout, _, K = w.shape
    p = (K - 1) * dil // 2
    xp = F.pad(x, (p, p))
    idx = torch.arange(T, device=x.device)[:, None] + dil * torch.arange(K, device=x.device)
    cols = xp[:, :, idx].permute(0, 2, 1, 3).reshape(B * T, Cin * K)
    y = _mm(cols, w.reshape(Cout, -1).t(), _mode(cls, Cin, Cout, K, dil, T)) + b
    return y.reshape(B, T, Cout).transpose(1, 2)


def _linear(rows, wb, cls):
    w, b = wb
    return _mm(rows, w.t(), _mode(cls, w.shape[1], w.shape[0], 1, 1, rows.shape[0])) + b


def head_ref(W, x, glob, cls=None):
    """CNNLSTM.forward (modules/quantize.py:106-125) on x [B][C][T] in x's dtype -> list of [B][T][out] ([B][out] when
    glob)."""
    B, Cn, T = x.shape
    f = aa_filter(x.dtype, x.device)
    h = x
    for j, d in enumerate((1, 2, 3)):
        u = W["units"][j]
        y = _conv(aa_act(h, f, *u["s1"]), u["c7"], d, cls)
        h = h + _conv(aa_act(y, f, *u["s2"]), u["c1"], 1, cls)
    h = aa_act(h, f, *W["final"]).transpose(1, 2)
    rows = h.mean(1) if glob else h.reshape(B * T, Cn)
    return [_linear(rows, wb, cls) if glob else _linear(rows, wb, cls).reshape(B, T, -1) for wb in W["heads"]]


def head_weights(sd, dtype=torch.float64, device="cpu"):
    """A CNNLSTM state_dict -> the restatement's weights (weight norm folded in float64, then cast to dtype)."""
    s = {k: v.to(device, torch.float64) for k, v in sd.items() if not k.endswith(".filter")}
    cast = lambda t: t.to(dtype)
    conv = lambda p: (cast(torch._weight_norm(s[p + ".weight_v"], s[p + ".weight_g"], 0)), cast(s[p + ".bias"]))
    act = lambda p: (cast(s[p + ".act.alpha"].reshape(-1)), cast(s[p + ".act.beta"].reshape(-1)))
    units = [{"s1": act(f"model.{j}.block.0"), "c7": conv(f"model.{j}.block.1"), "s2": act(f"model.{j}.block.2"),
              "c1": conv(f"model.{j}.block.3")} for j in range(3)]
    n = sum(1 for k in s if k.startswith("heads.") and k.endswith(".weight"))
    return {"units": units, "final": act("model.3"),
            "heads": [(cast(s[f"heads.{i}.weight"]), cast(s[f"heads.{i}.bias"])) for i in range(n)]}


FAP_USED = ("f0_predictor", "phone_predictor", "timbre_predictor", "rev_f0_predictor.1", "rev_content_predictor.1",
            "rev_timbre_predictor.1")


def fap_weights(sd, dtype=torch.float64, device="cpu"):
    """An FApredictors state_dict -> {part: head weights, or (w, b) of a plain linear} for the parts forward reads."""
    out = {}
    for name in FAP_USED:
        if name + ".weight" in sd:
            out[name] = tuple(sd[name + k].to(device, torch.float64).to(dtype) for k in (".weight", ".bias"))
        else:
            out[name] = head_weights({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")},
                                     dtype, device)
    return out


def fap_ref(Ws, lat, timbre, flags, timbre_norm, cls=None):
    """FApredictors.forward_v2 (modules/quantize.py:564-619, timbre_norm) or the four-latent forward (:507-563); the
    GradientReversal layers are identities and the latent sums accumulate into zeros_like, left to right."""
    f = flags
    head = lambda name, x, glob=False: head_ref(Ws[name], x, glob, cls)

    def total(terms):
        acc = torch.zeros_like(lat[0])
        for t in terms:
            acc = acc + t
        return acc
    if timbre_norm:
        p, c, r = lat[:3]
        content = head("phone_predictor", c)[0]
        spk = _linear(timbre, Ws["timbre_predictor"], cls)
        f0, uv = head("f0_predictor", p)
        pro = [c] * f["use_gr_content_f0"] + [r] * f["use_gr_residual_f0"]
        con = [p] * f["use_gr_prosody_phone"] + [r] * f["use_gr_residual_phone"]
        x_terms = [p, c, r]
    else:
        p, c, t, r = lat[:4]
        content = head("phone_predictor", c)[0]
        if f["norm_f0"]:
            spk = head("timbre_predictor", t, True)[0]
            f0, uv = head("f0_predictor", p)
        else:
            spk = head("timbre_predictor", total([t, p]), True)[0]
            f0, uv = head("f0_predictor", total([p, t]))
        pro = [c] * f["use_gr_content_f0"] + [t] * f["use_gr_timbre_prosody"] + [r] * f["use_gr_residual_f0"]
        con = [p] * f["use_gr_prosody_phone"] + [t] * f["use_gr_timbre_content"] + [r] * f["use_gr_residual_phone"]
        x_terms = [p, c, r] if f["norm_f0"] else [c, r]
    rev_f0, rev_uv = head("rev_f0_predictor.1", total(pro))
    rev_content = head("rev_content_predictor.1", total(con))[0]
    x_spk = head("rev_timbre_predictor.1", total(x_terms), True)[0] if f["use_gr_x_timbre"] else None
    return ({"f0": f0, "uv": uv, "content": content, "timbre": spk},
            {"rev_f0": rev_f0, "rev_uv": rev_uv, "rev_content": rev_content, "x_timbre": x_spk})


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatement against the oracle, and the separations the GPU bars rely on
# ---------------------------------------------------------------------------------------------------------------------
class _Float64Default:
    """The oracle builds its filter and zeros in the default dtype: float64 makes it the float64 twin."""

    def __enter__(self):
        self.prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.float64)

    def __exit__(self, *exc):
        torch.set_default_dtype(self.prev)


def _close(got, ref, tag):
    scale = max(ref.abs().max().item(), 1e-300)
    err = (got - ref).abs().max().item()
    assert err <= 1e-14 * scale, f"{tag}: {err:.3e} vs scale {scale:.3e}"


@pytest.mark.parametrize("T", [1, 2, 6, 7, 40])
def test_alias_free_reference_matches_the_oracle(T):
    """Both modes; T = 1 and 2 are shorter than the replicate pads."""
    from oracle import facodec_oracle as O
    _threads()
    g = torch.Generator().manual_seed(T)
    x = torch.randn(2, 5, T, generator=g, dtype=torch.float64)
    la, lb = torch.rand(5, generator=g, dtype=torch.float64) - 0.5, torch.rand(5, generator=g, dtype=torch.float64) - 0.5
    with _Float64Default():
        ri = O.alias_free_act(x, lambda u: u)
        rs = O.alias_free_act(x, lambda u: O.snake_beta(u, la, lb))
    f = aa_filter()
    _close(aa_act(x, f), ri, "identity")
    _close(aa_act(x, f, la, lb), rs, "snake")
    with _Float64Default():
        assert torch.equal(O.kaiser_sinc_filter1d(0.25, 0.3, 12).reshape(-1), f)


@pytest.mark.parametrize("indim,outdim,heads,glob,B,T", [(16, 3, 2, False, 2, 9), (32, 5, 1, True, 3, 4),
                                                         (16, 1, 1, True, 1, 1), (16, 7, 3, False, 2, 2)])
def test_head_reference_matches_the_oracle(indim, outdim, heads, glob, B, T):
    """T = 1, 2 and 4 are shorter than the dilation-2 and -3 pads."""
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    _threads()
    sd = synth.synth_cnnlstm(7 + T, indim, outdim, heads)
    x = torch.randn(B, indim, T, generator=torch.Generator().manual_seed(T), dtype=torch.float64)
    with _Float64Default(), torch.no_grad():
        ref = O.cnnlstm_forward({k: v.double() for k, v in sd.items()}, x, heads, global_pred=glob)
    got = head_ref(head_weights(sd), x, glob)
    assert len(got) == heads
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a.shape == b.shape
        _close(a, b, f"head {i}")


FAP_FLAG_SETS = {
    "build_model": dict(use_gr_content_f0=False, use_gr_prosody_phone=False, use_gr_residual_f0=True,
                        use_gr_residual_phone=True, use_gr_timbre_content=True, use_gr_timbre_prosody=False,
                        use_gr_x_timbre=True, norm_f0=True),
    "all": dict(use_gr_content_f0=True, use_gr_prosody_phone=True, use_gr_residual_f0=True, use_gr_residual_phone=True,
                use_gr_timbre_content=True, use_gr_timbre_prosody=True, use_gr_x_timbre=True, norm_f0=True),
    "none": dict(use_gr_content_f0=False, use_gr_prosody_phone=False, use_gr_residual_f0=False,
                 use_gr_residual_phone=False, use_gr_timbre_content=False, use_gr_timbre_prosody=False,
                 use_gr_x_timbre=False, norm_f0=True),
}


@pytest.mark.parametrize("timbre_norm,flag_set,norm_f0", [(True, "build_model", True), (True, "all", True),
                                                          (True, "none", True), (False, "build_model", True),
                                                          (False, "all", False), (False, "none", False),
                                                          (False, "all", True)])
def test_fa_predictors_reference_matches_the_oracle(timbre_norm, flag_set, norm_f0, built_lib):
    """Both forwards and every flag they branch on (zero, one, two and three summed latents; x_timbre on and off)."""
    import facodec_b200 as fb
    from oracle import facodec_oracle as O
    _threads()
    flags = dict(FAP_FLAG_SETS[flag_set], norm_f0=norm_f0)
    m = fb.FApredictors(in_dim=16, timbre_norm=timbre_norm, n_speakers=40, **flags).eval()
    sd = {k: v.double() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(3)
    lat = [torch.randn(2, 16, 6, generator=g, dtype=torch.float64) for _ in range(3 if timbre_norm else 4)]
    timbre = torch.randn(2, 16, generator=g, dtype=torch.float64)
    with _Float64Default(), torch.no_grad():
        ref = O.fa_predictors_forward(sd, lat, timbre if timbre_norm else None, timbre_norm=timbre_norm, **flags)
    got = fap_ref(fap_weights(sd), lat, timbre, flags, timbre_norm)
    for a, b in zip(got, ref):
        assert a.keys() == b.keys()
        for k in a:
            assert (a[k] is None) == (b[k] is None), k
            if a[k] is not None:
                _close(a[k], b[k], k)


def _head_refs(W64, W32, x, glob, fp32_ref=None):
    """{"64", "32", "bf16x3", "fp16"} outputs of one head (lists), as float64."""
    run32 = fp32_ref or (lambda fn, *a: fn(*a))
    with torch.no_grad():
        return {"64": head_ref(W64, x.double(), glob), "bf16x3": head_ref(W64, x.double(), glob, "bf16x3"),
                "fp16": head_ref(W64, x.double(), glob, "fp16"),
                "32": [y.double() for y in run32(head_ref, W32, x.float(), glob)]}


# (indim, outdim, heads, glob, B, T) of the CPU separation check
SEP_CASES = [(64, 1024, 1, False, 2, 40), (64, 20000, 1, True, 3, 20), (64, 1, 2, False, 2, 33), (16, 50, 1, False, 3, 9)]


@pytest.mark.parametrize("indim,outdim,heads,glob,B,T", SEP_CASES)
def test_bars_separate_the_classes(indim, outdim, heads, glob, B, T, built_lib):
    """For these seeds and shapes: the bf16x3 error is far above the F32 bar of the fp32-grade routes (max), the fp16
    error is far above the default route's F_BF16 bar (max), and its rms is 16x the bf16x3 one or more, so the 1/8 bar
    leaves twice the bf16x3 class's rms."""
    import facodec_b200 as fb
    _threads()
    m = fb.CNNLSTM(indim, outdim, heads, global_pred=glob, seed=9)
    sd = m.state_dict()
    x = torch.randn(B, indim, T, generator=torch.Generator().manual_seed(T))
    r = _head_refs(head_weights(sd), head_weights(sd, torch.float32), x, glob)
    for i in range(heads):
        y64 = r["64"][i]
        scale = y64.abs().max().item()
        e32, eb, eh = ((r[k][i] - y64).abs().max().item() for k in ("32", "bf16x3", "fp16"))
        rb, rh = _rms(r["bf16x3"][i] - y64), _rms(r["fp16"][i] - y64)
        print(f"SEP {indim}->{outdim} glob={glob} B={B} T={T} head {i}: max f32 {e32:.3e} bf16x3 {eb:.3e} fp16 {eh:.3e} "
              f"(bf16x3 x{eb / (F32 * e32 + C * scale):.1f} the F32 bar, fp16 x{eh / (F_BF16 * eb + C * scale):.1f} the "
              f"F_BF16 bar)  rms fp16/bf16x3 {rh / rb:.1f}")
        assert eb >= 1.15 * (F32 * e32 + C * scale)
        assert eh >= 1.15 * (F_BF16 * eb + C * scale)
        assert rh >= 16 * rb


# ---------------------------------------------------------------------------------------------------------------------
# GPU: Activation1d (alias_free_act_kernel)
# ---------------------------------------------------------------------------------------------------------------------
def _fp32_ref(fn, *a):
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return fn(*a)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32


def _with_options(eng, opts, fn):
    try:
        for k, v in opts.items():
            eng.set_option(k, v)
        return fn()
    finally:
        for k in opts:
            eng.set_option(k, OPTION_DEFAULTS[k])


_ACTS = {}


def _act(C=None, la=None, lb=None):
    """One Activation1d per channel count (identity when C is None), its log-scale alpha / beta set to la / lb."""
    import facodec_b200 as fb
    if C not in _ACTS:
        _ACTS[C] = fb.Activation1d(identity=True) if C is None else fb.Activation1d(C, alpha_logscale=True)
    m = _ACTS[C]
    if C is not None:
        with torch.no_grad():
            m.alpha.copy_(la)
            m.beta.copy_(lb)
    return m


def identity_bound(x64):
    """The a-priori elementwise bound on |y - y64| of the identity mode (module docstring)."""
    f = aa_filter(device=x64.device)
    F1 = f.abs().sum().item()
    S = max(f[0::2].abs().sum().item(), f[1::2].abs().sum().item())
    g = lambda n: n * U32 / (1 - n * U32)
    T = x64.shape[-1]
    Xw = _clamped(x64.abs(), -6, T + 12, T).unfold(-1, 13, 1).amax(-1)
    k = (g(12) + U32) * (1 + 10 * U32) + g(6) * (1 + U32) + U32 + 64 * 2.0 ** -53
    return 2 * F1 * S * k * Xw


AA_T = [1, 2, 3, 5, 6, 7, 11, 12, 13, 255, 256, 257, 511, 512, 513, 2000]
AA_CASES = [(8, 1, T) for T in AA_T] + [(5, 3, T) for T in AA_T] + [(2, 1024, T) for T in AA_T] + \
           [(70, 1024, 7), (8, 1024, 320)]
# log-parameter regimes of SnakeBeta: as synth.synth_cnnlstm makes them (|log a|, |log b| <= 0.3), log a = +2 (arguments
# in the tens), log b = -3 (the sin^2 term x 20), and the synthetic ones on inputs x 8
AA_REGIMES = ("synth", "log_alpha_2", "log_beta_m3", "x8")


def _aa_inputs(B, Cn, T, regime, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cn, T, generator=g)
    la = (torch.rand(Cn, generator=g) * 2 - 1) * 0.3
    lb = (torch.rand(Cn, generator=g) * 2 - 1) * 0.3
    if regime == "log_alpha_2":
        la = torch.full_like(la, 2.0)
    elif regime == "log_beta_m3":
        lb = torch.full_like(lb, -3.0)
    elif regime == "x8":
        x = x * 8
    return x, la, lb


def check_snake(tag, y, x, la, lb):
    xd = x.cuda()
    with torch.no_grad():
        y64 = aa_act(xd.double(), aa_filter(device="cuda"), la.double().cuda(), lb.double().cuda())
    y32 = _fp32_ref(aa_act, xd, aa_filter(torch.float32, "cuda"), la.cuda(), lb.cuda()).double()
    err, err32, scale = (y.double() - y64).abs().max().item(), (y32 - y64).abs().max().item(), y64.abs().max().item()
    bar = F32 * err32 + C * scale
    print(f"AA {tag}: max|y-y64| {err:.3e}  max|y32-y64| {err32:.3e}  err/err32 {err / max(err32, 1e-300):.2f}  "
          f"err/bar {err / bar:.3f}  scale {scale:.2f}")
    assert err <= bar, f"{tag}: max|y - y64| = {err:.3e} > {bar:.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("B,Cn,T", AA_CASES)
def test_alias_free_act_vs_fp64(B, Cn, T, built_lib):
    """Identity mode elementwise under the a-priori bound; SnakeBeta (synthetic log-parameters) under the fp32 bar."""
    x, la, lb = _aa_inputs(B, Cn, T, "synth", 100 * Cn + T)
    xd = x.cuda()
    y = _act()(xd)
    torch.cuda.synchronize()
    with torch.no_grad():
        y64 = aa_act(xd.double(), aa_filter(device="cuda"))
    d = (y.double() - y64).abs()
    bound = identity_bound(xd.double())
    print(f"AA identity B={B} C={Cn} T={T}: max err/bound {(d / bound).max().item():.3f}")
    assert torch.isfinite(y).all() and (d <= bound).all(), \
        f"identity: {int((d > bound).sum())} samples over the a-priori bound, worst at {int((d - bound).argmax())}"
    check_snake(f"synth B={B} C={Cn} T={T}", _act(Cn, la, lb)(xd), x, la, lb)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", AA_REGIMES[1:])
@pytest.mark.parametrize("B,Cn,T", [(5, 3, 13), (2, 1024, 257), (8, 1024, 320)])
def test_alias_free_act_regimes(regime, B, Cn, T, built_lib):
    x, la, lb = _aa_inputs(B, Cn, T, regime, 7 * T + Cn)
    check_snake(f"{regime} B={B} C={Cn} T={T}", _act(Cn, la, lb)(x.cuda()), x, la, lb)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 2, 7, 256, 257, 2000])
def test_alias_free_act_constant_rows(T, built_lib):
    """A row holding one constant comes back as that constant at every sample, both ends included, within 8 ulp."""
    g = torch.Generator().manual_seed(T)
    Cn = 16
    c = torch.randn(3, Cn, 1, generator=g) * torch.pow(2.0, torch.randint(-20, 20, (3, Cn, 1), generator=g).float())
    cd = c.cuda()
    y = _act()(cd.expand(3, Cn, T).contiguous())
    torch.cuda.synchronize()
    ulps = (y - cd).abs() / torch.pow(2.0, torch.floor(torch.log2(cd.abs())) - 23)
    print(f"CONST T={T}: worst {ulps.max().item():.2f} ulp")
    assert (ulps <= 8).all(), f"{int((ulps > 8).sum())} samples more than 8 ulp off, worst at {int(ulps.argmax())}"


@pytest.mark.gpu
def test_alias_free_act_channels_follow_their_parameters(built_lib):
    """Channel c uses alpha[c] and beta[c]: permuting the channels with their parameters permutes the output bit for bit."""
    import facodec_b200 as fb
    Cn = 1024
    x, la, lb = _aa_inputs(2, Cn, 300, "synth", 5)
    perm = torch.randperm(Cn, generator=torch.Generator().manual_seed(6))
    y = _act(Cn, la, lb)(x.cuda()).clone()
    m2 = fb.Activation1d(Cn, alpha_logscale=True)
    with torch.no_grad():
        m2.alpha.copy_(la[perm])
        m2.beta.copy_(lb[perm])
    y2 = m2(x[:, perm].contiguous().cuda())
    torch.cuda.synchronize()
    assert torch.equal(y2, y[:, perm.cuda()])
    assert not torch.equal(y2, y)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: one head through fac_head_forward
# ---------------------------------------------------------------------------------------------------------------------
_HEADS = {}


def _head(indim, outdim, heads, glob):
    """One CNNLSTM per geometry (its own synthetic weights) with its float64 / float32 reference weights on the GPU."""
    import facodec_b200 as fb
    key = (indim, outdim, heads, glob)
    if key not in _HEADS:
        if len(_HEADS) >= 4:
            _HEADS.pop(next(iter(_HEADS)))
        m = fb.CNNLSTM(indim, outdim, heads, global_pred=glob, seed=indim % 7).eval()
        sd = m.state_dict()
        _HEADS[key] = (m, {"64": head_weights(sd, torch.float64, "cuda"), "32": head_weights(sd, torch.float32, "cuda")})
    return _HEADS[key]


def check_output(tag, y, refs, factor, indim):
    """One output tensor against its references {"64", "32", "bf16x3", "fp16"} under the route's bars; returns the
    bars it breaks (every output of a call is measured before the test fails)."""
    if not torch.isfinite(y).all():
        return [f"{tag}: non-finite output"]
    y64 = refs["64"]
    assert y.shape == y64.shape, tag
    d = y.double() - y64
    err, scale = d.abs().max().item(), y64.abs().max().item()
    wide = indim == 1024
    rk, rh = _rms(d), _rms(refs["fp16"] - y64)
    fma_only = rh == 0                   # no layer of this output on the tensor cores: the fp32 bar on every route
    if factor is None and not fma_only:
        eref = (refs["bf16x3"] - y64).abs().max().item()
        bar, what = (F_BF16_1024 if wide else F_BF16) * eref + C * scale, "bf16x3"
    else:
        factor = F32 if factor is None else factor
        eref = (refs["32"] - y64).abs().max().item()
        if wide:
            factor = {F32: F32_1024, F_TF32X3_TRUNC: F_TF32X3_TRUNC_1024}[factor]
        bar, what = factor * eref + C * scale, "f32"
    rbar = RMS_FP16_1024 if wide else 1 / 8
    print(f"HEAD {tag}: max|y-y64| {err:.3e}  max|y_{what}-y64| {eref:.3e}  err/err_{what} {err / max(eref, 1e-300):.2f}  "
          f"err/bar {err / bar:.3f}  rms(y-y64)/rms(y_fp16-y64) {rk / max(rh, 1e-300):.4f}  scale {scale:.3f}")
    fails = []
    if not err <= bar:
        fails.append(f"{tag}: max|y - y64| = {err:.3e} > {bar:.3e}")
    if not fma_only and not rk <= rh * rbar:
        fails.append(f"{tag}: rms(y - y64) = {rk:.3e} > {rbar} x {rh:.3e} (one-pass fp16 class)")
    return fails


HEAD_CASES = [(64, 50, 2, False, 3, T) for T in (1, 2, 9, 10, 63, 64, 65)] + \
             [(16, 1, 8, True, B, T) for B, T in ((3, 10), (8, 65))] + [(16, 1024, 2, True, 1, 1)] + \
             [(16, 1024, 1, False, 8, 9), (16, 50, 1, True, 3, 2)] + \
             [(64, 1024, 1, False, 1, T) for T in (127, 128, 129)] + [(64, 1024, 1, False, 3, 43)] + \
             [(64, 20000, 1, True, 3, 10), (1024, 1, 2, False, 3, 64), (1024, 50, 2, True, 3, 63),
              (1024, 1024, 1, False, 1, 321), (1024, 20000, 1, True, 1, 2), (1024, 20000, 1, True, 8, 320)]


@pytest.mark.gpu
@pytest.mark.parametrize("indim,outdim,heads,glob,B,T", HEAD_CASES)
def test_head_vs_fp64(indim, outdim, heads, glob, B, T, built_lib):
    """Every output of one CNNLSTM on every route against the float64 restatement."""
    m, W = _head(indim, outdim, heads, glob)
    x = torch.randn(B, indim, T, generator=torch.Generator().manual_seed(B * 1000 + T)).cuda()
    refs = _head_refs(W["64"], W["32"], x, glob, _fp32_ref)
    fails = []
    for route, (opts, factor) in ROUTES.items():
        outs = _with_options(m._engine, opts, lambda: m(x))
        torch.cuda.synchronize()
        for i, y in enumerate(outs):
            fails += check_output(f"{route} {indim}->{outdim} glob={glob} B={B} T={T} head {i}", y,
                                  {k: v[i] for k, v in refs.items()}, factor, indim)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("indim,outdim,rows", [(16, 1, 3), (64, 50, 129), (64, 1024, 129), (1024, 20000, 8)])
def test_head_linear_vs_fp64(indim, outdim, rows, built_lib):
    """The linear kind of fac_head_finalize (_HeadLinear: FApredictors.timbre_predictor under timbre_norm)."""
    from facodec_b200.modules import _HeadLinear
    m = _HeadLinear(indim, outdim, seed=indim)
    x = torch.randn(rows, indim, generator=torch.Generator().manual_seed(rows)).cuda()
    wb64 = (m.weight.detach().cuda().double(), m.bias.detach().cuda().double())
    wb32 = tuple(t.float() for t in wb64)
    with torch.no_grad():
        refs = {"64": _linear(x.double(), wb64, None), "bf16x3": _linear(x.double(), wb64, "bf16x3"),
                "fp16": _linear(x.double(), wb64, "fp16"), "32": _fp32_ref(_linear, x, wb32, None).double()}
    fails = []
    for route, (opts, factor) in ROUTES.items():
        y = _with_options(m._engine, opts, lambda: m(x))
        torch.cuda.synchronize()
        fails += check_output(f"{route} linear {indim}->{outdim} rows={rows}", y, refs, factor, indim)
    assert not fails, "\n".join(fails)


PROP_CASES = [(64, 1024, 1, False, 3, 65), (1024, 20000, 1, True, 3, 43), (16, 50, 2, True, 3, 10),
              (64, 1, 8, False, 4, 9)]


@pytest.mark.gpu
@pytest.mark.parametrize("indim,outdim,heads,glob,B,T", PROP_CASES)
def test_head_exact_properties(indim, outdim, heads, glob, B, T, built_lib):
    """Batch invariance (default and FMA routes), repeatability, and options that must not move a bit: tensor_cores 1
    (heads are not upstream of the VQ), decoder_conv7_fp16 0 (heads have no one-pass blob), tc_occ2_maxn 128 (same N)."""
    m, _ = _head(indim, outdim, heads, glob)
    x = torch.randn(B, indim, T, generator=torch.Generator().manual_seed(T)).cuda()
    run = lambda opts, xx=x: [y.clone() for y in _with_options(m._engine, opts, lambda: m(xx))]
    for opts in ({}, {"tensor_cores": 0}):
        full = run(opts)
        for b in range(B):
            one = run(opts, x[b:b + 1].contiguous())
            for i in range(heads):
                assert torch.equal(one[i][0], full[i][b]), f"{opts} utterance {b} head {i}: batch-variant"
    ref = run({})
    torch.cuda.synchronize()
    for opts in ({}, {"tensor_cores": 1}, {"decoder_conv7_fp16": 0}, {"tc_occ2_maxn": 128}):
        got = run(opts)
        torch.cuda.synchronize()
        for i in range(heads):
            assert torch.equal(got[i], ref[i]), f"{opts or 'second call'}: head {i} differs"


@pytest.mark.gpu
@pytest.mark.parametrize("indim,outdim,heads,glob,B,T", [(1024, 20000, 1, True, 3, 43), (64, 50, 2, False, 3, 65),
                                                         (16, 1, 8, True, 2, 5)])
def test_head_outputs_stay_in_their_views(indim, outdim, heads, glob, B, T, built_lib):
    """fac_head_forward writing into views of NaN-filled buffers: every output element comes back finite and equal to a
    plain call's, and the guard regions before and after it come back unchanged."""
    m, _ = _head(indim, outdim, heads, glob)
    x = torch.randn(B, indim, T, generator=torch.Generator().manual_seed(3)).cuda()
    plain = [y.clone() for y in m(x)]
    n = B * outdim if glob else B * T * outdim
    G = 1024
    bufs = [torch.full((G + n + G,), float("nan"), device="cuda") for _ in range(heads)]
    before = [b.view(torch.int32).clone() for b in bufs]
    arr = (ctypes.c_void_p * heads)(*[b[G:].data_ptr() for b in bufs])
    e = m._engine
    rc = e.L.fac_head_forward(e.handle, m._head_id, _p(x), B, T, arr, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    for i, b in enumerate(bufs):
        out = b[G:G + n]
        assert torch.isfinite(out).all(), f"head {i}: {int((~torch.isfinite(out)).sum())} outputs not written"
        assert torch.equal(out, plain[i].reshape(-1))
        w = b.view(torch.int32)
        assert torch.equal(w[:G], before[i][:G]) and torch.equal(w[G + n:], before[i][G + n:]), f"head {i}: guard written"


@pytest.mark.gpu
@pytest.mark.parametrize("indim,outdim,heads,glob", [(64, 1024, 1, False), (64, 20000, 1, True)])
def test_head_workspace_poison(indim, outdim, heads, glob, built_lib):
    """A larger call with NaN inputs first leaves NaN across the engine's workspace; the real call is then finite and
    bit-identical to the same call on a fresh engine."""
    import facodec_b200 as fb
    m, _ = _head(indim, outdim, heads, glob)
    m(torch.full((4, indim, 200), float("nan"), device="cuda"))
    x = torch.randn(3, indim, 65, generator=torch.Generator().manual_seed(65)).cuda()
    got = [y.clone() for y in m(x)]
    fresh = fb.CNNLSTM(indim, outdim, heads, global_pred=glob, seed=1).eval()
    fresh.load_state_dict(m.state_dict())
    want = fresh(x)
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert torch.isfinite(a).all() and torch.equal(a, b)


@pytest.mark.gpu
def test_head_errors(built_lib):
    import facodec_b200 as fb
    x = torch.randn(1, 24, 5, device="cuda")
    with pytest.raises(fb.FacError, match="multiple of 16"):
        fb.CNNLSTM(24, 4, 1).eval()(x)
    x = torch.randn(1, 16, 5, device="cuda")
    for outdim, heads in ((4, 0), (4, 9), (0, 1)):
        with pytest.raises(fb.FacError):
            fb.CNNLSTM(16, outdim, heads).eval()(x)
    e = fb.modules.Engine()
    e._ensure(torch.device("cuda"))
    hid = e.L.fac_head_begin(e.handle)
    assert hid >= 0
    out = torch.full((1, 5, 4), float("nan"), device="cuda")
    arr = (ctypes.c_void_p * 1)(out.data_ptr())
    assert e.L.fac_head_forward(e.handle, hid, _p(x), 1, 5, arr, None) == FAC_ERR_STATE       # nothing finalized
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: FApredictors
# ---------------------------------------------------------------------------------------------------------------------
def _latents(B, T, indim, n, seed):
    """n latents [B][indim][T] at the quantizer's output scale: sums of out_proj(codebook[random code]) over the prosody
    (1), content (2) and residual (3) quantizers of the synthetic FAquantizer (the fourth, timbre-like latent of the
    four-latent forward reuses the residual form), cut to indim channels."""
    from conftest import state_dicts
    from oracle import facodec_oracle as O
    sd = state_dicts(0)["quantizer"]
    g = torch.Generator().manual_seed(seed)
    out = []
    for name, nq in (("prosody", 1), ("content", 2), ("residual", 3), ("residual", 3))[:n]:
        z = torch.zeros(B, 1024, T)
        for q in range(nq):
            p = f"{name}_quantizer.quantizers.{q}"
            cb = sd[p + ".codebook.weight"][torch.randint(0, 1024, (B, T), generator=g)]          # [B][T][8]
            w = O._wn_weight(sd, p + ".out_proj").reshape(1024, 8)
            z = z + (cb @ w.t() + sd[p + ".out_proj.bias"]).transpose(1, 2)
        out.append(z[:, :indim].contiguous())
    return out


def _fap_check(tag, got, refs, factor, indim):
    fails = []
    for part in range(2):
        for k, y in got[part].items():
            r = {c: refs[c][part][k] for c in refs}
            if y is None:
                assert r["64"] is None, k
                continue
            fails += check_output(f"{tag} {k}", y, r, factor, indim)
    return fails


def _fap_refs(Ws, lat, timbre, flags, timbre_norm):
    cuda = [t.cuda() for t in lat]
    tv = timbre.cuda() if timbre is not None else None
    with torch.no_grad():
        d = lambda cls: fap_ref(Ws["64"], [t.double() for t in cuda], tv.double() if tv is not None else None, flags,
                                timbre_norm, cls)
        refs = {"64": d(None), "bf16x3": d("bf16x3"), "fp16": d("fp16")}
    p32 = _fp32_ref(fap_ref, Ws["32"], cuda, tv, flags, timbre_norm)
    refs["32"] = tuple({k: (v.double() if v is not None else None) for k, v in part.items()} for part in p32)
    return refs


@pytest.mark.gpu
def test_fa_predictors_training_geometry(built_lib):
    """build_model(with_predictors=True).fa_predictors (forward_v2, the flags of modules/commons.py:311-322) at 8 x 4 s
    (B = 8, T = 320, in_dim = 1024) on the default route: what bench.py --workload trainfwd runs every step."""
    import facodec_b200 as fb
    m = fb.build_model(with_predictors=True).fa_predictors.eval()
    assert m.flags["timbre_norm"] and m.in_dim == 1024
    sd = m.state_dict()
    Ws = {"64": fap_weights(sd, torch.float64, "cuda"), "32": fap_weights(sd, torch.float32, "cuda")}
    lat = _latents(8, 320, 1024, 3, 21)
    timbre = torch.randn(8, 1024, generator=torch.Generator().manual_seed(22))
    got = m([t.cuda() for t in lat], timbre.cuda())
    torch.cuda.synchronize()
    refs = _fap_refs(Ws, lat, timbre, m.flags, True)
    fails = _fap_check("default fa_predictors B=8 T=320", got, refs, None, 1024)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("norm_f0", [True, False])
def test_fa_predictors_four_latents(norm_f0, built_lib):
    """The four-latent forward (timbre_norm = False) at in_dim 256 on every route."""
    import facodec_b200 as fb
    flags = dict(FAP_FLAG_SETS["all"], norm_f0=norm_f0)
    m = fb.FApredictors(in_dim=256, timbre_norm=False, **flags).eval()
    sd = m.state_dict()
    Ws = {"64": fap_weights(sd, torch.float64, "cuda"), "32": fap_weights(sd, torch.float32, "cuda")}
    lat = _latents(3, 50, 256, 4, 23)
    refs = _fap_refs(Ws, lat, None, m.flags, False)
    fails = []
    for route, (opts, factor) in ROUTES.items():
        got = _with_options(m._engine, opts, lambda: m([t.cuda() for t in lat]))
        torch.cuda.synchronize()
        fails += _fap_check(f"{route} four latents norm_f0={norm_f0}", got, refs, factor, 256)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 255, 256, 257, 148 * 16 * 256 + 5])
def test_add3_is_torch_fp32_left_to_right(n, built_lib):
    """fac_add3 = (a + b) + c in fp32, bit for bit (the reference's zeros_like accumulation gives the same bits), and
    a + b without c; n past the kernel's grid-stride cap included."""
    import facodec_b200 as fb
    e = fb.modules.Engine()
    e._ensure(torch.device("cuda"))
    g = torch.Generator().manual_seed(n)
    a, b, c = (torch.randn(n, generator=g) * torch.pow(2.0, torch.randint(-12, 12, (n,), generator=g).float())
               for _ in range(3))
    a, b, c = a.cuda(), b.cuda(), c.cuda()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for terms in ((a, b, c), (a, b)):
        out = torch.full_like(a, float("nan"))
        rc = e.L.fac_add3(e.handle, _p(terms[0]), _p(terms[1]), _p(terms[2]) if len(terms) > 2 else None, n, _p(out), st)
        assert rc == 0
        want = torch.zeros_like(a)
        for t in terms:
            want = want + t
        torch.cuda.synchronize()
        assert torch.equal(out, want)
