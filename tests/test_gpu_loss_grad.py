"""Gradients of the dac/nn/loss.py criteria (facodec_b200.losses MultiScaleSTFTLoss / MelSpectrogramLoss / L1Loss through
torch autograd: fac_spectral_loss_grad / fac_l1_loss_grad) against torch autograd of the oracle restatements on the CPU.

Reference gradients: the restatement evaluated in float64 (Hann window and STFT in float64, the librosa filterbank the
library uses -- rounded to fp32 -- cast to float64).  Error bar, self-calibrating: per case, the normwise relative error
||g - g64|| / ||g64|| of every utterance's GPU gradient must be at most 4 x the largest such error of the same restatement
run in float32 on the CPU (torch autograd over pocketfft), + 1e-6, + two explicit terms for what fp32 spectra cannot
decide (below).  The float32 yardstick is large where the loss itself is ill-conditioned:
d log10(clamp(|X|)^2) / d|X| = 2 / (|X| ln 10) amplifies rounding in near-silent bins, and an L1 sign taken on a near-tie
flips with the rounding.

The gradient GEMM's operands.  dL/dspec carries the loss's 1 / N mean factor (1e-9 ... 1e-6 at the benchmark shape), below
fp16's normal range, and the promoted GEMM class splits its activations into fp16 hi + 2^11-scaled fp16 lo without a
scale of its own; the gradient kernel therefore scales each row by a power of two (largest entry in [2^13, 2^14)) and
the overlap-add undoes it, both exactly.  With that, the mel criteria meet the 4x bar at every shape here, the bench
batch (32, 96 000) included, with no allowance for the GEMM.

The two terms, each per utterance and signal:
  * ties (_tie_allowance): where x's and y's mel band / magnitude agree within 2^-20 relative, the L1 subgradient's sign
    is not determined by fp32 spectra, and either sign is a valid subgradient.  The term is the largest change a flipped
    sign there can make.  Measured on an H100: MelSpectrogramLoss() at (32, 96 000), utterance 13, w = 2048 frame 173
    band 14 (vx = 0.22403718, vy = 0.22403724 in float64): the GPU takes the other sign, and its dx / dy errors
    (8.30e-3 / 7.49e-3) equal this term; every other utterance is within 5e-5.
  * near-silent STFT bins (_class_allowance, MultiScaleSTFTLoss only): the forward DFT GEMM's products carry 22
    significant bits, against the float32 FFT's 24 over log2(w) stages, and the log term's gradient amplifies a
    magnitude error by 1 / |X|.  Measured: at (3, 1025), dy of utterance 1 is off by 1.24e-2 (fp32: 7.7e-5) through one
    bin, w = 2048 frame 0 bin 291, |Y| = 2.37e-4 in float64, whose gradient 2 / (|Y| ln 10) / N = 0.40 per unit
    dominates; the deviation is 2.6 % of that bin's gradient.  The term is the first-order effect of a random-walk
    magnitude error 2^-22 sqrt(sum_n (win_n x_n)^2) over the bins, times 4.
The loss value itself uses the same spectrum (bit-identical to the no-grad call), so the gradient is that of the value
the library returns.

Exact properties: the loss value with gradients requested is the no-grad value bit for bit; two calls give bit-identical
gradients; identical inputs give an all-zero gradient (sgn(0) = 0); a pair silent below clamp_eps gives a zero log-term
gradient; L1's dL/dy is -dL/dx bit for bit; gradients of a weighted sum of criteria are the weighted sum of gradients.
"""
import contextlib
import ctypes
import math
import types

import pytest
import torch
import torch.nn.functional as F

WINDOWS_TRAIN = [32, 64, 128, 256, 512, 1024, 2048]
CRITERIA = {
    # train.py:155-163
    "mel_train": dict(kind="mel", n_mels=[5, 10, 20, 40, 80, 160, 320], window_lengths=WINDOWS_TRAIN, mel_fmin=[0.0] * 7,
                      mel_fmax=[None] * 7, pow=1.0, mag_weight=0.0, log_weight=1.0, clamp_eps=1e-5),
    "mel_default": dict(kind="mel", n_mels=[150, 80], window_lengths=[2048, 512], mel_fmin=[0.0, 0.0], mel_fmax=[None, None],
                        pow=2.0, mag_weight=1.0, log_weight=1.0, clamp_eps=1e-5),
    "stft_default": dict(kind="stft", window_lengths=[2048, 512], pow=2.0, mag_weight=1.0, log_weight=1.0, clamp_eps=1e-5),
    "l1": dict(kind="l1"),
}
# the bench.py batch, 4 s utterances, ragged, shortest legal for w = 2048 (T = w / 2 + 1)
SHAPES = [(32, 96000), (4, 96000), (2, 5001), (3, 1025)]
WANTS = {"x": (True, False), "y": (False, True), "both": (True, True)}
SR = 24000


@contextlib.contextmanager
def _default_dtype(dt):
    old = torch.get_default_dtype()
    torch.set_default_dtype(dt)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


def _criterion(name):
    from facodec_b200 import losses
    c = dict(CRITERIA[name])
    kind = c.pop("kind")
    if kind == "l1":
        return losses.L1Loss()
    if kind == "stft":
        return losses.MultiScaleSTFTLoss(**c)
    return losses.MelSpectrogramLoss(**c)


def _oracle_loss(name, x, y):
    """The oracle restatement (oracle/facodec_oracle.py) in x's dtype: window, STFT and filterbank in that dtype."""
    from oracle import facodec_oracle as O
    c = CRITERIA[name]
    if c["kind"] == "l1":
        return F.l1_loss(x, y)
    mag = O._audiotools_magnitude
    with _default_dtype(x.dtype):                    # torch.hann_window inside the oracle follows the default dtype
        loss = 0.0
        if c["kind"] == "stft":                      # O.multiscale_stft_loss with the magnitude chosen above
            for w in c["window_lengths"]:
                mx, my = mag(x, w), mag(y, w)
                loss = loss + c["log_weight"] * F.l1_loss(mx.clamp(c["clamp_eps"]).pow(c["pow"]).log10(),
                                                          my.clamp(c["clamp_eps"]).pow(c["pow"]).log10())
                loss = loss + c["mag_weight"] * F.l1_loss(mx, my)
            return loss
        for nm, f0, f1, w in zip(c["n_mels"], c["mel_fmin"], c["mel_fmax"], c["window_lengths"]):
            basis = O.librosa_mel_filters(SR, w, nm, f0, f1).to(x.dtype)      # fp32 weights (as the library), cast
            mx = (mag(x, w).transpose(2, -1) @ basis.T).transpose(-1, 2)
            my = (mag(y, w).transpose(2, -1) @ basis.T).transpose(-1, 2)
            loss = loss + c["log_weight"] * F.l1_loss(mx.clamp(c["clamp_eps"]).pow(c["pow"]).log10(),
                                                      my.clamp(c["clamp_eps"]).pow(c["pow"]).log10())
            loss = loss + c["mag_weight"] * F.l1_loss(mx, my)
        return loss


TIE = 2.0 ** -20          # |vx - vy| <= TIE * max(vx, vy): a tie within the spectra's fp32 evaluation error


def _tie_loss(name, x, y):
    """float64: the part of the loss carried by the bands / bins where x's and y's values (mel bands or magnitudes) tie
    within TIE, each taken with sign +1: sum over them of (log_weight * (log10(clamp(vx)^pow) + log10(clamp(vy)^pow))
    + mag_weight * (vx + vy)) / N.  At such a tie the L1 subgradient's sign is not determined by fp32 spectra: an
    implementation may take either sign, which moves its gradient by up to twice this term's gradient."""
    from oracle import facodec_oracle as O
    c = CRITERIA[name]
    if c["kind"] == "l1":
        return None
    loss, any_tie = 0.0, False
    with _default_dtype(x.dtype):
        for i, w in enumerate(c["window_lengths"]):
            mx, my = O._audiotools_magnitude(x, w), O._audiotools_magnitude(y, w)
            if c["kind"] == "mel":
                basis = O.librosa_mel_filters(SR, w, c["n_mels"][i], c["mel_fmin"][i], c["mel_fmax"][i]).to(x.dtype)
                mx = (mx.transpose(2, -1) @ basis.T).transpose(-1, 2)
                my = (my.transpose(2, -1) @ basis.T).transpose(-1, 2)
            tie = ((mx - my).abs() <= TIE * torch.maximum(mx, my)).detach()
            if not tie.any():
                continue
            any_tie = True
            lg = lambda v: v.clamp(c["clamp_eps"]).pow(c["pow"]).log10()
            per = c["log_weight"] * (lg(mx) + lg(my)) + c["mag_weight"] * (mx + my)
            loss = loss + (per * tie).sum() / mx.numel()
    return loss if any_tie else None


def _tie_allowance(name, x, y, g64):
    """Per utterance and signal: 2 ||d(tie loss)/d.|| / ||g64||, the largest gradient change a different sign choice at
    the ties (_tie_loss) can make, relative to the reference gradient's norm."""
    a = x.detach().double().clone().requires_grad_(True)
    b = y.detach().double().clone().requires_grad_(True)
    lt = _tie_loss(name, a, b)
    if lt is None:
        return [0.0] * x.shape[0], [0.0] * x.shape[0]
    ga, gb = torch.autograd.grad(lt, (a, b))
    out = []
    for g, ref in ((ga, g64[0]), (gb, g64[1])):
        n = g.reshape(g.shape[0], -1).norm(dim=1) / ref.reshape(ref.shape[0], -1).norm(dim=1)
        out.append([2.0 * float(v) for v in n])
    return tuple(out)


def _cpu_grads(name, x, y, dtype):
    a = x.detach().to(dtype).clone().requires_grad_(True)
    b = y.detach().to(dtype).clone().requires_grad_(True)
    _oracle_loss(name, a, b).backward()
    return a.grad.double(), b.grad.double()


def _relerr(g, ref):
    """Per-utterance normwise relative error; g, ref [B, ...]."""
    g, ref = g.double().reshape(g.shape[0], -1), ref.double().reshape(ref.shape[0], -1)
    return ((g - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-300)).tolist()


U22 = 2.0 ** -22


def _class_allowance(name, sig, g64):
    """Per utterance, the normwise relative gradient error the forward DFT GEMM's precision class explains in near-silent
    STFT bins (module docstring): per bin, the first-order change of its log-term gradient log_weight * pow / (N |X| ln 10)
    under a magnitude error of the class's random-walk scale e = 2^-22 sqrt(sum_n (win_n x_n)^2), times the norm
    sqrt(sum win^2) of the bin's DFT row, root-sum-squared over bins and scales (independent errors), times 4 (the factor
    the bar gives the float32 yardstick).  0 for the mel criteria (a band sums many bins) and for L1."""
    c = CRITERIA[name]
    if c["kind"] != "stft":
        return [0.0] * sig.shape[0]
    extra = torch.zeros(sig.shape[0], dtype=torch.float64)
    s64 = sig[:, 0].double()
    for w in c["window_lengths"]:
        win = torch.hann_window(w, periodic=True, dtype=torch.float64)
        X = torch.stft(s64, w, w // 4, window=win, return_complex=True, center=True).abs()          # [B, nb, F]
        fr = F.pad(s64[:, None], (w // 2, w // 2), mode="reflect")[:, 0].unfold(-1, w, w // 4)      # [B, F, w]
        e = U22 * (fr * win).pow(2).sum(-1).sqrt()                                                  # [B, F]
        per_bin = c["log_weight"] * c["pow"] / (X.numel() * math.log(10)) * e[:, None, :] / X.clamp_min(c["clamp_eps"]) ** 2
        extra += per_bin.pow(2).sum(dim=(1, 2)) * float(win.pow(2).sum())
    norms = g64.reshape(g64.shape[0], -1).norm(dim=1)
    return [4.0 * float(a.sqrt() / n) for a, n in zip(extra, norms)]


_REF = {}


def _reference(name, B, T):
    """(x, y, (gx64, gy64), (err32 of dx, err32 of dy), (class allowance of dx, of dy)) for one criterion and shape,
    cached across the wanted-input cases."""
    key = (name, B, T)
    if key not in _REF:
        from facodec_b200 import synth
        x, y = synth.synth_loss_pair(B, T, seed=9)          # [B, 1, T], as the oracle takes them
        g64 = _cpu_grads(name, x, y, torch.float64)
        g32 = _cpu_grads(name, x, y, torch.float32)
        err32 = tuple(max(_relerr(a, b)) for a, b in zip(g32, g64))
        ties = _tie_allowance(name, x, y, g64)
        allow = tuple([cl + ti for cl, ti in zip(_class_allowance(name, sig, g), tie)] for sig, g, tie in zip((x, y), g64, ties))
        _REF.clear()
        _REF[key] = (x, y, g64, err32, allow)
    return _REF[key]


def _gpu(name, x, y, want_x, want_y):
    crit = _criterion(name)
    a = x.detach().cuda().requires_grad_(want_x)
    b = y.detach().cuda().requires_grad_(want_y)
    loss = crit(a, b)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), (a.grad if want_x else None), (b.grad if want_y else None)


def _bar_check(tag, g, ref, err32, allow):
    errs = _relerr(g.cpu(), ref)
    bars = [4.0 * err32 + 1e-6 + a for a in allow]
    print(f"LOSSGRAD {tag}: gpu err {max(errs):.3e}  fp32 cpu err {err32:.3e}  allowance {max(allow):.3e}  "
          f"worst err / bar {max(e / b for e, b in zip(errs, bars)):.3f}")
    if any(e > b for e, b in zip(errs, bars)):
        # locate the worst samples for the report
        d = (g.cpu().double() - ref).abs()
        idx = torch.topk(d.flatten(), 5).indices
        worst = [(int(i) // d.shape[-1], int(i) % d.shape[-1], float(d.flatten()[i]), float(ref.flatten()[i])) for i in idx]
        pytest.fail(f"{tag}: per-utterance errors {errs} over the bars {bars}; worst (b, t, |diff|, ref): {worst}")


@pytest.mark.gpu
@pytest.mark.parametrize("want", list(WANTS))
@pytest.mark.parametrize("B,T", SHAPES)
@pytest.mark.parametrize("name", list(CRITERIA))
def test_gradient_vs_fp64_autograd(built_lib, name, B, T, want):
    import warnings
    warnings.simplefilter("ignore")
    x, y, (gx64, gy64), (ex32, ey32), (ax, ay) = _reference(name, B, T)
    want_x, want_y = WANTS[want]
    loss, gx, gy = _gpu(name, x, y, want_x, want_y)
    with torch.no_grad():
        loss_nograd = _criterion(name)(x.cuda(), y.cuda())
    torch.cuda.synchronize()
    assert torch.equal(loss.reshape(()), loss_nograd.reshape(())), (float(loss), float(loss_nograd))
    tag = f"{name} B={B} T={T} want={want}"
    if want_x:
        assert gx.shape == x.shape and gx.dtype == torch.float32
        _bar_check(tag + " dx", gx, gx64, ex32, ax)
    if want_y:
        assert gy.shape == y.shape and gy.dtype == torch.float32
        _bar_check(tag + " dy", gy, gy64, ey32, ay)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CRITERIA))
def test_gradients_bit_reproducible(built_lib, name):
    from facodec_b200 import synth
    x, y = synth.synth_loss_pair(3, 24000, seed=4)
    r1 = _gpu(name, x[:, 0], y[:, 0], True, True)
    r2 = _gpu(name, x[:, 0], y[:, 0], True, True)
    for a, b in zip(r1, r2):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CRITERIA))
def test_identical_inputs_give_zero_gradient(built_lib, name):
    from facodec_b200 import synth
    x, _ = synth.synth_loss_pair(2, 12000, seed=6)
    x = x[:, 0]
    _, gx, gy = _gpu(name, x, x.clone(), True, True)
    assert not gx.any() and not gy.any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mel_default", "stft_default"])
def test_silent_pair_has_zero_log_gradient(built_lib, name):
    """|X| <= w * 1e-9 < clamp_eps everywhere: the clamp passes no gradient, so with mag_weight = 0 the gradient is 0; with
    the magnitude term it is that term's alone (compared with a criterion whose log_weight is 0)."""
    from facodec_b200 import losses, synth
    x, y = synth.synth_loss_pair(2, 8000, seed=3)
    x, y = (x[:, 0] * 1e-9).cuda(), (y[:, 0] * 1e-9).cuda()
    c = dict(CRITERIA[name])
    kind = c.pop("kind")
    cls = losses.MelSpectrogramLoss if kind == "mel" else losses.MultiScaleSTFTLoss

    def grad(**over):
        a = x.clone().requires_grad_(True)
        cls(**{**c, **over})(a, y).backward()
        return a.grad

    assert not grad(mag_weight=0.0).any()
    g_all, g_mag = grad(), grad(log_weight=0.0)
    assert g_mag.abs().max() > 0
    assert torch.equal(g_all, g_mag)


@pytest.mark.gpu
def test_l1_dy_is_minus_dx(built_lib):
    from facodec_b200 import synth
    x, y = synth.synth_loss_pair(2, 5001, seed=2)
    x, y = x[:, 0], y[:, 0].clone()
    y[0, :100] = x[0, :100]                         # ties: sgn(0) = 0 on both sides
    _, gx, gy = _gpu("l1", x, y, True, True)
    assert torch.equal(gy, -gx)
    assert not gx[0, :100].any()
    assert (gx[0, 100:].abs() == gx.abs().max()).all()


@pytest.mark.gpu
def test_weighted_sum_backward(built_lib):
    """(15 * mel(x, y) + l1(x, y)).backward() = 15 g_mel + g_l1 (train.py:357 weights the mel term 15)."""
    from facodec_b200 import synth
    x, y = synth.synth_loss_pair(2, 24000, seed=8)
    x, y = x[:, 0].cuda(), y[:, 0].cuda()
    mel, l1 = _criterion("mel_train"), _criterion("l1")
    a = x.clone().requires_grad_(True)
    (15 * mel(a, y) + l1(a, y)).backward()
    a1 = x.clone().requires_grad_(True)
    mel(a1, y).backward()
    a2 = x.clone().requires_grad_(True)
    l1(a2, y).backward()
    expect = 15 * a1.grad + a2.grad
    assert torch.allclose(a.grad, expect, rtol=1e-6, atol=1e-12 * float(expect.abs().max()))


@pytest.mark.gpu
def test_conv_weight_gradient_through_audio_signal(built_lib):
    """train.py wraps pred_wave in AudioSignal(pred_wave, 24000): gradients reach a conv that made pred_wave through
    .audio_data ([B, 1, T]) and the criterion's [B, 1, T] -> [B, T] view.  Two checks: dL/dpred against the fp64
    oracle gradient within the module's bar (4 x the fp32 CPU error + 1e-6, + the tie term), and the conv's weight and
    bias gradients against the fp64 chain rule applied to that GPU dL/dpred (the conv's backward, fp32 on the GPU)."""
    from facodec_b200 import synth
    wave, target = synth.synth_loss_pair(2, 24000, seed=12)

    def run(device, dtype, loss_fn):
        torch.manual_seed(0)
        conv = torch.nn.Conv1d(1, 1, 7, padding=3).to(device=device, dtype=dtype)
        pred = conv(wave.to(device=device, dtype=dtype))
        pred.retain_grad()
        loss = loss_fn(pred, target.to(device=device, dtype=dtype))
        if loss is None:
            return None, None
        loss.backward()
        return pred.grad.double().cpu(), torch.cat([conv.weight.grad.flatten(), conv.bias.grad.flatten()]).double().cpu()

    sig = lambda t: types.SimpleNamespace(audio_data=t, sample_rate=SR)
    gp, gw = run("cuda", torch.float32, lambda p, t: _criterion("mel_train")(sig(p), sig(t)))
    gp64, _ = run("cpu", torch.float64, lambda p, t: _oracle_loss("mel_train", p, t))
    gp32, _ = run("cpu", torch.float32, lambda p, t: _oracle_loss("mel_train", p, t))
    gpt, _ = run("cpu", torch.float64, lambda p, t: _tie_loss("mel_train", p, t))
    err32 = max(_relerr(gp32, gp64))
    allow = [0.0] * gp.shape[0] if gpt is None else _relerr(2 * gpt + gp64, gp64)
    _bar_check("conv dL/dpred", gp, gp64, err32, allow)
    # the chain rule in fp64 on the GPU's dL/dpred: dW[k] = sum_t g[t] * wave_padded[t + k], db = sum_t g[t]
    wpad = F.pad(wave.double(), (3, 3))
    ref_w = torch.stack([(gp * wpad[..., k:k + wave.shape[-1]]).sum() for k in range(7)] + [gp.sum()])
    assert float((gw - ref_w).norm() / ref_w.norm()) <= 1e-5, (gw, ref_w)


@pytest.mark.gpu
def test_error_paths(built_lib):
    import facodec_b200 as fb
    from facodec_b200 import synth
    x, y = synth.synth_loss_pair(1, 4000, seed=1)
    mel = _criterion("mel_default")
    with pytest.raises(fb.FacError):
        mel(x.clone().requires_grad_(True), y.cuda())              # CPU tensor: no fallback
    with pytest.raises(fb.FacError):
        mel(x.cuda().requires_grad_(True), y.cuda()[..., :3000])
    with pytest.raises(fb.FacError):
        _criterion("l1")(x.cuda().requires_grad_(True), y.cuda()[..., :3000])
    a = x.cuda().requires_grad_(True)
    g, = torch.autograd.grad(mel(a, y.cuda()), a, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()                                         # once_differentiable: no second order


def test_criteria_to_returns_self():
    """train.py:154-164 builds each criterion with .to(device)."""
    for name in CRITERIA:
        c = _criterion(name)
        assert c.to("cuda") is c
        assert c.to(torch.device("cuda", 0), non_blocking=True) is c


def test_transposed_dft_plans(built_lib):
    """The gradient GEMM dframes = dspec basis^T is a K = 1 "conv" with Cin = ld (2 * (w / 2 + 1) rounded up to 128) and
    Cout = w: the tensor-core kernel plans it for every window 16 ... 4096 in the promoted classes (3xTF32 split and fp16
    hi + scaled lo), so it never falls back to the fp32 FMA conv."""
    from facodec_b200 import _lib
    L = _lib.load()
    for k in range(4, 13):
        w = 1 << k
        ld = (2 * (w // 2 + 1) + 127) // 128 * 128
        for mode in (1, 3):
            out = (ctypes.c_int * 8)()
            assert L.fac_debug_tc_plan(ld, w, 1, 1, 1, 4096, mode, 0, out) == 0, (w, mode)
            assert w % out[0] == 0 and out[0] > 0
