"""The loss kernels frame by frame against float64: fac_reconstruction_loss (losses.py:65-89) and fac_spectral_loss /
fac_l1_loss (dac/nn/loss.py criteria), through the per-scale taps recon.{dft,terms,fb}.<i> / spec.{dft,terms,fb}.<i>.

What is checked, per scale, against references built on the CPU in float64:
  * the host-built filterbanks (HTK: torchaudio.functional.melscale_fbanks in float64; Slaney: the oracle's librosa
    restatement before it rounds), weight by weight;
  * the DFT rows of both signals (stft_frames_kernel + the K = 1 GEMM on the promoted tensor-core class, or on the fp32
    SIMT conv with tensor_cores = 0), element by element against torch.stft, padding columns exactly zero;
  * the per-frame terms (mel_loss_terms_kernel / spec_loss_terms_kernel), first from the tapped DFT rows and filterbank
    (so the bound measures the terms kernel alone), then from float64 x and y with the DFT bound carried through;
  * the fixed-order fp64 sums (strided_sum_kernel, sqdiff_partial_kernel, absdiff_partial_kernel) and the fp32 combines.
Both tensor-core settings run (tensor_cores = 2: promoted fp16 hi + scaled-lo class; 0: conv_cl_kernel).

Bounds (u = 2^-24; gamma_n(v) = n v / (1 - n v), Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., 3.1:
a sum whose terms each pass through at most n roundings of unit v is within gamma_n(v) sum |terms| of the exact one).
CUDA's single-precision functions have these maximum errors (CUDA C++ Programming Guide, "Single-Precision
Floating-Point Functions"): logf 1 ulp, log10f 2 ulp, powf 4 ulp, sqrtf correctly rounded; 1 ulp <= 2u |result|.
  * Filterbank.  The host evaluates the same fp64 formula and rounds once: |fb - ref| <= 2u |ref| plus the fp64 noise
    of a weight whose bin lies on a breakpoint (both sides compute the ramps from breakpoints that carry fp64 rounding,
    a few ulps of the Nyquist frequency: delta_f = 64 * 2^-53 * (sr / 2)): norm_m * 2 delta_f / (smallest gap of band m).
    A bin further than delta_f outside a triangle must hold exactly 0 (empty bands, triangle edges, fmin / fmax).
  * DFT.  Each output is one dot over the s (or w) windowed samples against a basis rounded once to fp32 (u |w_n|).
    Promoted tensor-core class: both operands split into fp16 hi + 2^11-scaled fp16 lo (22 significant bits, the dropped
    lo * lo product ~2^-22), windows of <= 48 chained MMAs added into an fp32 master: gamma_s(2^-22).  SIMT: an fp32 FMA
    chain, gamma_s(u).  So |dRe|, |dIm| <= e = (c + u) sum_n |w_n x_n|, c = gamma_s(2^-22) or gamma_s(u).
  * Per-frame terms, from DFT values with error e per element:
      power P = Re^2 + Im^2 (one FMA + one product): |dP| <= 2 sqrt2 |X| e + 2 e^2 + gamma_2 P; magnitude
      |d|X|| <= sqrt2 e + gamma_3 |X|;
      mel sums of nonnegative terms: the reconstruction kernel runs 4 FMA chains of ceil(nb / 4) and 2 adds
      (gamma_{ceil(nb/4)+4} with the power's two roundings), the spectral kernel 2 chains of ceil(nb / 2) and 1 add;
      log(|S| + eps): the add rounds (u), |d log v| <= dv / (v - dv) for the input error dv, + 1 ulp;
      clamp(v, eps): |d clamp(v)| <= |dv|; v^pow: p dv / (v - dv) relative, + the rounding of pow (none for pow = 1,
      u for the product of pow = 2, 4 ulp for powf); log10: the relative error r becomes r / ((1 - r) ln 10), + 2 ulp;
      the per-frame sums: 64 values through a 6-level tree (reconstruction) / ceil(n_out / 128) sequential adds, a
      5-level warp tree and 2 adds (spectral), each value first formed by one subtraction;
      sqrt(v / 64): the division is exact, |d sqrt(v)| <= min(sqrt(dv), dv / sqrt(v)), + u.
  * Sums.  strided_sum adds the fp32 frame terms in fp64 (relative error ~1e-13) and the combine rounds once to fp32,
    so every returned component is within 1 fp32 ulp of the fp64 sum of the tapped frame terms times its factor.  The
    mse and the L1 loss round 1024 fp64 block partials to fp32 first (u each, nonnegative) and the result once more:
    |got - ref| <= 2u ref (+ the fp64 noise).
  * The reconstruction loss is the fp32 combine of the returned components, bit for bit.  nvcc contracts a * b + c to
    one FMA (--fmad=true), so loss_combine_kernel computes fma(100, mse, fma(a_0, l2_0, l1_0)), then + fma(a_i, l2_i,
    l1_i) for i = 1..5 (a_i = sqrtf(s_i / 2)), and spec_loss_combine_kernel L = fma(v_mag_i, mw, fma(v_log_i, lw, L)).

Mutations (test_mutants_are_seen): reference variants a subtly wrong kernel could compute -- a frame shifted by one
sample, zero or replicate padding instead of reflect, a symmetric Hann window, the last frame dropped, one filterbank
band shifted by one bin, eps = 1e-5 instead of 1e-7 (reconstruction), pow ignored (spectral), and the DFT of the first
and last frame of every utterance 2 % too large.  Each one is seen by the elementwise bounds here.  Measured on the
benchmark shape (B = 4, T = 96000, scale s = 64: 6001 frames per utterance), the scalar tolerance of
test_gpu_losses.py (2e-5 relative per component) misses only the 2 % edge-frame error (l1_64 moves by ~1.6e-5, l2_64
not at all); on these white-noise signals the other variants move l1_64 or l2_64 by 2.5e-5 (band shift) to 1.6e-2
(symmetric window), so the scalar tests would see them too.  test_scalar_misses_claim_cpu checks this list.
"""
import contextlib
import ctypes
import math
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24
U22 = 2.0 ** -22
LN10 = math.log(10.0)
ULP_LOGF, ULP_LOG10F, ULP_POWF = 1, 2, 4
EPS_RECON = float(np.float32(1e-7))          # the kernel's eps (fp32)
SCALAR_REL = 2e-5                             # test_gpu_losses.py's tolerance on the reconstruction components


def gamma(n, u=U):
    return n * u / (1 - n * u)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _cdiv(a, b):
    return -(-a // b)


def _ratio(err, bound):
    """max err / bound, 0 / 0 counted as 0."""
    r = torch.where(bound > 0, err / bound, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.max()) if r.numel() else 0.0


def _check(tag, err, bound):
    r = _ratio(err, bound)
    print(f"LOSSERR {tag} max err/bound={r:.3e} maxerr={float(err.max()) if err.numel() else 0.0:.3e}")
    assert (err <= bound).all(), f"{tag}: max err/bound {r:.3f}"
    return r


# ---------------------------------------------------------------------------------------------------------------------
# exact fp32 arithmetic (for the combine kernels)
# ---------------------------------------------------------------------------------------------------------------------
def _rn32(q):
    """Round the exact rational q to the nearest fp32 (ties to even)."""
    f = np.float32(float(q))
    best = f
    for c in (np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))):
        dc, db = abs(Fraction(float(c)) - q), abs(Fraction(float(best)) - q)
        if dc < db or (dc == db and int(np.float32(c).view(np.uint32)) % 2 == 0):
            best = c
    return np.float32(best)


def _fma32(a, b, c):
    return _rn32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _recon_combine(t):
    """loss_combine_kernel as compiled (module docstring) on the 13 returned fp32 components."""
    t = [np.float32(v) for v in t]
    a = [np.sqrt(np.float32(64 << i) * np.float32(0.5)) for i in range(6)]
    L = _fma32(t[0], np.float32(100), _fma32(t[2], a[0], t[1]))
    for i in range(1, 6):
        L = np.float32(L + _fma32(t[2 + 2 * i], a[i], t[1 + 2 * i]))
    return L


def _spec_combine(v_mag, v_log, mag_weight, log_weight):
    L = np.float32(0)
    for m, lg in zip(v_mag, v_log):
        L = _fma32(np.float32(lg), np.float32(log_weight), L)
        L = _fma32(np.float32(m), np.float32(mag_weight), L)
    return L


def _ulp32(v):
    return float(np.spacing(np.abs(np.float32(v))))


# ---------------------------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------------------------
def _hann(n, periodic=True):
    return torch.hann_window(n, periodic=periodic, dtype=torch.float64)


def _stft64(w, n_fft, win_len, window=None, pad_mode="reflect"):
    """[N, T] float64 -> [N * F, n_fft // 2 + 1] complex rows (frame-major per signal), torch.stft(center=True)."""
    win = _hann(win_len) if window is None else window
    X = torch.stft(w, n_fft, hop_length=win_len // 4, win_length=win_len, window=win, center=True, pad_mode=pad_mode,
                   normalized=False, onesided=True, return_complex=True)
    return X.transpose(1, 2).reshape(-1, n_fft // 2 + 1)


def _sabs(w, win_len):
    """sum_n |w_n x_n| of every frame, [N * F] (the window's nonzero span is win_len samples centred on f * hop)."""
    p = win_len // 2
    xp = F.pad(w[:, None], (p, p), mode="reflect")[:, 0]
    fr = xp.unfold(1, win_len, win_len // 4)
    return (fr.abs() * _hann(win_len)).sum(-1).reshape(-1)


def _dft_coef(win_len, tc):
    return (gamma(win_len, U22) if tc else gamma(win_len)) + U


def _htk_fb64(nb):
    """torchaudio.functional.melscale_fbanks(nb, 0, 8000, 64, 16000, norm=None, 'htk') in float64, its breakpoints, norm."""
    import torchaudio
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        fb = torchaudio.functional.melscale_fbanks(nb, 0.0, 8000.0, 64, 16000, None, "htk")
    finally:
        torch.set_default_dtype(old)
    hz2mel = lambda f: 2595.0 * np.log10(1.0 + f / 700.0)
    mel2hz = lambda m: 700.0 * (10.0 ** (m / 2595.0) - 1.0)
    bp = mel2hz(np.linspace(hz2mel(0.0), hz2mel(8000.0), 66))
    return fb.double(), torch.from_numpy(bp), torch.ones(64, dtype=torch.float64), torch.linspace(0, 8000, nb, dtype=torch.float64)


def _slaney_fb64(sr, n_fft, n_mels, fmin, fmax):
    from oracle import facodec_oracle as O
    fmax = sr / 2.0 if fmax is None else float(fmax)
    fb = O.librosa_mel_filters(sr, n_fft, n_mels, fmin, fmax, dtype=torch.float64).T.contiguous()
    f_sp, min_log_hz = 200.0 / 3.0, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    hz2mel = lambda f: min_log_mel + np.log(f / min_log_hz) / logstep if f >= min_log_hz else f / f_sp
    mel2hz = lambda m: np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)
    bp = torch.from_numpy(mel2hz(np.linspace(hz2mel(float(fmin)), hz2mel(fmax), n_mels + 2)))
    norm = 2.0 / (bp[2:] - bp[:-2])
    return fb, bp, norm, torch.linspace(0, sr / 2.0, n_fft // 2 + 1, dtype=torch.float64)


def _fb_bound(fb64, bp, norm, freqs):
    """(bound, outside): 2u |w| + the breakpoint noise per weight; the bins further than delta_f outside each triangle."""
    df = 64 * 2.0 ** -53 * float(freqs[-1])
    gap = torch.minimum(bp[1:-1] - bp[:-2], bp[2:] - bp[1:-1])
    outside = (freqs[:, None] <= bp[None, :-2] - df) | (freqs[:, None] >= bp[None, 2:] + df)
    return 2 * U * fb64.abs() + (norm * 2 * df / gap)[None, :], outside


def _check_fb(tag, got, fb64, bp, norm, freqs):
    """got [nb][n_out] (the tap) against the fp64 formula: zeros outside the triangles, 2u + breakpoint noise inside."""
    got = got.double()
    bound, outside = _fb_bound(fb64, bp, norm, freqs)
    assert (fb64[outside] == 0).all()
    assert (got[outside] == 0).all(), f"{tag}: nonzero weight outside its triangle"
    return _check(tag, (got - fb64).abs(), bound)


def _recon_terms(re, im, e, fb, B, Fr, eps=EPS_RECON):
    """mel_loss_terms_kernel in float64 with its bounds: rows [2 B Fr][nb] (x, then G_x), e [2 B Fr] the rows' DFT error
    bound (0 for the tapped rows).  Returns (t1, e1, t2, e2), each [B Fr]."""
    nb = fb.shape[0]
    P = re * re + im * im
    e = e[:, None]
    eP = 2 * math.sqrt(2) * P.sqrt() * e + 2 * e * e
    mel = P @ fb
    emel = eP @ fb + gamma(_cdiv(nb, 4) + 4) * ((P + eP) @ fb)
    n = B * Fr
    sx, sg, ex, eg = mel[:n], mel[n:], emel[:n], emel[n:]
    t1 = (sx - sg).abs().sum(1)
    e1 = gamma(7) * ((sx - sg).abs() + ex + eg).sum(1) + (ex + eg).sum(1)

    def lg(s, es):
        v = s + eps
        dv = es + U * (v + es)
        rel = torch.where(v > dv, dv / (v - dv), torch.full_like(v, math.inf))
        lv = v.log()
        return lv, rel + 2 * U * ULP_LOGF * (lv.abs() + rel)

    lx, elx = lg(sx, ex)
    lgg, elg = lg(sg, eg)
    dl = lx - lgg
    edl = elx + elg + U * (dl.abs() + elx + elg)
    d2 = (dl * dl).sum(1)
    ed2 = (2 * dl.abs() * edl + edl * edl + U * (dl.abs() + edl) ** 2).sum(1) + gamma(6) * ((dl.abs() + edl) ** 2).sum(1)
    t2 = (d2 / 64).sqrt()
    q = ed2 / 64
    et2 = torch.minimum(q.sqrt(), torch.where(d2 > 0, q / t2.clamp_min(1e-300), torch.full_like(q, math.inf)))
    return t1, e1, t2, et2 + U * (t2 + q.sqrt())


def _spec_terms(re, im, e, fb, B, Fr, eps, pw):
    """spec_loss_terms_kernel in float64 with its bounds (fb [nb][n_out] or None)."""
    eps = float(np.float32(eps))
    mag = (re * re + im * im).sqrt()
    e = e[:, None]
    emag = math.sqrt(2) * e + gamma(3) * (mag + math.sqrt(2) * e)
    if fb is not None:
        nb = fb.shape[0]
        v = mag @ fb
        ev = emag @ fb + gamma(_cdiv(nb, 2) + 2) * ((mag + emag) @ fb)
    else:
        v, ev = mag, emag
    depth = _cdiv(v.shape[1], 128) + 8
    n = B * Fr
    vx, vy, ex, ey = v[:n], v[n:], ev[:n], ev[n:]
    t1 = (vx - vy).abs().sum(1)
    e1 = gamma(depth) * ((vx - vy).abs() + ex + ey).sum(1) + (ex + ey).sum(1)
    r_pow = 0.0 if pw == 1.0 else (U if pw == 2.0 else 2 * ULP_POWF * U)

    def lg(val, ev_):
        c = val.clamp_min(eps)
        rel = torch.where(c > ev_, pw * ev_ / (c - ev_), torch.full_like(c, math.inf)) + r_pow
        L = pw * c.log10()
        el = torch.where(rel < 1, rel / ((1 - rel) * LN10), torch.full_like(rel, math.inf))
        return L, el + 2 * U * ULP_LOG10F * (L.abs() + el)

    Lx, elx = lg(vx, ex)
    Ly, ely = lg(vy, ey)
    t2 = (Lx - Ly).abs().sum(1)
    e2 = gamma(depth) * ((Lx - Ly).abs() + elx + ely).sum(1) + (elx + ely).sum(1)
    return t1, e1, t2, e2


# ---------------------------------------------------------------------------------------------------------------------
# running the kernels with taps
# ---------------------------------------------------------------------------------------------------------------------
def _engine():
    from facodec_b200 import losses
    return losses._engine(torch.device("cuda:0"))


@contextlib.contextmanager
def _tensor_cores(e, v):
    e.set_option("tensor_cores", v)
    try:
        yield
    finally:
        e.set_option("tensor_cores", 2)


def _with_taps(e, sizes, fn):
    bufs = {k: torch.full((n,), float("nan"), device="cuda") for k, n in sizes.items()}
    try:
        for k, t in bufs.items():
            assert e.L.fac_debug_tap(e.handle, k.encode(), _p(t), t.numel()) == 0
        out = fn()
        torch.cuda.synchronize()
    finally:
        for k in bufs:
            e.L.fac_debug_tap(e.handle, k.encode(), None, 0)
    return out, {k: t.cpu() for k, t in bufs.items()}


def _recon_geom(i):
    s = 64 << i
    n_fft = max(s, 512)
    nb = n_fft // 2 + 1
    return s, n_fft, nb, (2 * nb + 127) // 128 * 128


def _spec_geom(w):
    nb = w // 2 + 1
    return nb, (2 * nb + 127) // 128 * 128


def _run_recon(x, g, tc):
    from facodec_b200 import losses
    e = _engine()
    B, T = x.shape
    sizes = {}
    for i in range(6):
        s, _, nb, ld = _recon_geom(i)
        Fr = T // (s // 4) + 1
        sizes[f"recon.dft.{i}"] = 2 * B * Fr * ld
        sizes[f"recon.terms.{i}"] = B * Fr * 2
        sizes[f"recon.fb.{i}"] = nb * 64
    with _tensor_cores(e, tc):
        (L, terms), taps = _with_taps(e, sizes, lambda: losses.reconstruction_loss(x.cuda(), g.cuda(), return_terms=True))
    return L.cpu(), terms.cpu(), taps


def _spec_cfg_geom(cfg, T):
    out = []
    for i, w in enumerate(cfg["windows"]):
        nb, ld = _spec_geom(w)
        nm = cfg["n_mels"][i] if cfg.get("n_mels") else 0
        out.append((w, nb, ld, T // (w // 4) + 1, nm))
    return out


def _spec_module(cfg):
    from facodec_b200 import losses
    kw = dict(window_lengths=cfg["windows"], clamp_eps=cfg.get("eps", 1e-5), mag_weight=cfg.get("mw", 1.0),
              log_weight=cfg.get("lw", 1.0), pow=cfg.get("pow", 2.0), sample_rate=cfg.get("sr", 24000))
    if cfg.get("n_mels"):
        return losses.MelSpectrogramLoss(n_mels=cfg["n_mels"], mel_fmin=cfg["fmin"], mel_fmax=cfg["fmax"], **kw)
    return losses.MultiScaleSTFTLoss(**kw)


def _run_spec(cfg, x, y, tc):
    e = _engine()
    B, T = x.shape
    sizes = {}
    for i, (w, nb, ld, Fr, nm) in enumerate(_spec_cfg_geom(cfg, T)):
        sizes[f"spec.dft.{i}"] = 2 * B * Fr * ld
        sizes[f"spec.terms.{i}"] = B * Fr * 2
        if nm:
            sizes[f"spec.fb.{i}"] = nb * nm
    mod = _spec_module(cfg)
    with _tensor_cores(e, tc):
        L, taps = _with_taps(e, sizes, lambda: mod(x.cuda(), y.cuda()))
    return L.cpu(), taps


def _split_rows(buf, rows, ld, nb):
    got = buf.view(rows, ld).double()
    return got[:, 0:2 * nb:2], got[:, 1:2 * nb:2], got[:, 2 * nb:]


def _check_dft(tag, buf, X, sabs, c, B, Fr, nb, ld):
    re, im, pad = _split_rows(buf, 2 * B * Fr, ld, nb)
    assert (pad == 0).all(), f"{tag}: padding columns beyond 2 nb are not zero"
    bound = (c * sabs)[:, None].expand_as(re)
    err = torch.maximum((re - X.real).abs(), (im - X.imag).abs())
    edge = torch.tensor([j * Fr + f for j in range(2 * B) for f in (0, Fr - 1)])
    _check(tag + " edge frames", err[edge], bound[edge])
    return _check(tag, err, bound), re, im


# ---------------------------------------------------------------------------------------------------------------------
# signals
# ---------------------------------------------------------------------------------------------------------------------
def _pair(B, T, seed):
    from facodec_b200 import synth
    x, g = synth.synth_loss_pair(B, T, seed=seed)
    return x[:, 0].contiguous(), g[:, 0].contiguous()


def _silent_pair(T=6000):
    """Utterance 0 silent at its start and in the middle, utterance 1 silent at its end (in both signals at the edges,
    only in x in the middle): frames of exact zeros, so the l2 term sees log(eps)."""
    x, g = _pair(2, T, 21)
    x[0, :700] = 0
    g[0, :700] = 0
    x[0, 3000:4000] = 0
    x[1, -900:] = 0
    g[1, -900:] = 0
    return x, g


RECON_CASES = {
    "b1_t1025": lambda: _pair(1, 1025, 3),
    "b3_t30011": lambda: _pair(3, 30011, 4),
    "b4_t96000": lambda: _pair(4, 96000, 5),
    "b34_t1100": lambda: _pair(34, 1100, 6),
    "silent": _silent_pair,
    "x_eq_g": lambda: (_pair(2, 3000, 7)[0],) * 2,
}


def _recon_reference(x64, g64, i):
    """Per scale i: fp64 DFT rows, their per-frame bound factor sum |w x| and the fp64 HTK filterbank."""
    s, n_fft, nb, ld = _recon_geom(i)
    w2 = torch.cat([x64, g64])
    return _stft64(w2, n_fft, s), _sabs(w2, s), _htk_fb64(nb)


# ---------------------------------------------------------------------------------------------------------------------
# reconstruction loss
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc", [2, 0])
@pytest.mark.parametrize("case", list(RECON_CASES))
def test_reconstruction_loss_per_frame(case, tc, built_lib):
    x, g = RECON_CASES[case]()
    B, T = x.shape
    L, terms, taps = _run_recon(x, g, tc)
    L2, terms2, _ = _run_recon(x, g, tc)
    assert torch.equal(L, L2) and torch.equal(terms, terms2), "two calls differ"
    x64, g64 = x.double(), g.double()
    tag = f"recon {case} tc={tc}"
    mse = float(((x64 - g64) ** 2).mean())
    _check(tag + " mse", torch.tensor([abs(float(terms[0]) - mse)]), torch.tensor([2 * U * mse * (1 + 1e-9) + 1e-300]))
    for i in range(6):
        s, n_fft, nb, ld = _recon_geom(i)
        Fr = T // (s // 4) + 1
        X, sabs, (fb64, bp, norm, freqs) = _recon_reference(x64, g64, i)
        fb = taps[f"recon.fb.{i}"].view(nb, 64).double()
        _check_fb(f"{tag} s={s} fb", fb, fb64, bp, norm, freqs)
        c = _dft_coef(s, tc == 2)
        _, re, im = _check_dft(f"{tag} s={s} dft", taps[f"recon.dft.{i}"], X, sabs, c, B, Fr, nb, ld)
        tr = taps[f"recon.terms.{i}"].view(B * Fr, 2).double()
        # the terms kernel alone: from the tapped rows and filterbank
        t1, e1, t2, e2 = _recon_terms(re, im, torch.zeros(2 * B * Fr, dtype=torch.float64), fb, B, Fr)
        _check(f"{tag} s={s} terms.l1", (tr[:, 0] - t1).abs(), e1)
        _check(f"{tag} s={s} terms.l2", (tr[:, 1] - t2).abs(), e2)
        # the whole chain from fp64 x and G_x
        t1c, e1c, t2c, e2c = _recon_terms(X.real, X.imag, c * sabs, fb, B, Fr)
        _check(f"{tag} s={s} chain.l1", (tr[:, 0] - t1c).abs(), e1c)
        _check(f"{tag} s={s} chain.l2", (tr[:, 1] - t2c).abs(), e2c)
        # the fixed-order sums: 1 ulp of the fp64 sum of the tapped frame terms
        l1 = float(tr[:, 0].sum()) / (B * Fr * 64.0)
        l2 = float(tr[:, 1].sum()) / (B * Fr)
        for k, ref in ((1 + 2 * i, l1), (2 + 2 * i, l2)):
            _check(f"{tag} s={s} sum{k}", torch.tensor([abs(float(terms[k]) - ref)]), torch.tensor([_ulp32(ref)]))
        if case == "x_eq_g":
            assert (tr == 0).all()
    if case == "x_eq_g":
        assert (terms == 0).all() and float(L) == 0.0
    assert np.float32(L.item()) == _recon_combine(terms.numpy()), (float(L), float(_recon_combine(terms.numpy())))


# ---------------------------------------------------------------------------------------------------------------------
# spectral losses
# ---------------------------------------------------------------------------------------------------------------------
SPEC_CASES = {
    # every window length at the shortest legal T of the largest (T = 4096 / 2 + 1), pow = 2, both terms
    "stft_all_windows": (dict(windows=[16, 32, 64, 128, 256, 512, 1024, 2048, 4096]), 2, 2049),
    # HTK-free Slaney banks: 1 band, fmin > 0 / fmax < sr / 2, 150 bands, 1024 bands over 2049 bins; pow = 1, no mag term
    "mel_44k": (dict(windows=[2048, 512, 4096, 64], n_mels=[1, 5, 150, 1024], fmin=[0.0, 50.0, 0.0, 300.0],
                     fmax=[None, 7000.0, None, 10000.0], pow=1.0, mw=0.0, sr=44100), 2, 128 * 40 + 1),
    # more mels than bins (320 bands over 17 bins), pow = 0.5, no log term; T = k hop - 1
    "mel_16k": (dict(windows=[32, 2048], n_mels=[320, 80], fmin=[0.0, 0.0], fmax=[None, None], pow=0.5, lw=0.0,
                     sr=16000), 3, 512 * 10 - 1),
    # the training defaults (150 / 80 bands over 2048 / 512, pow 2, 24 kHz) at T = k hop + 1
    "mel_defaults": (dict(windows=[2048, 512], n_mels=[150, 80], fmin=[0.0, 0.0], fmax=[None, None]), 2, 512 * 30 + 1),
    # the shortest legal T of a single small window, and train.py's 7-scale mel loss at 24 kHz
    "stft_w16_short": (dict(windows=[16]), 3, 9),
    "mel_train": (dict(windows=[32, 64, 128, 256, 512, 1024, 2048], n_mels=[5, 10, 20, 40, 80, 160, 320],
                       fmin=[0.0] * 7, fmax=[None] * 7, pow=1.0, mw=0.0), 2, 5001),
}


def _spec_reference(cfg, x64, y64, i, w):
    w2 = torch.cat([x64, y64])
    nm = cfg["n_mels"][i] if cfg.get("n_mels") else 0
    fbr = _slaney_fb64(cfg.get("sr", 24000), w, nm, cfg["fmin"][i], cfg["fmax"][i]) if nm else None
    return _stft64(w2, w, w), _sabs(w2, w), fbr


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [2, 0])
@pytest.mark.parametrize("case", list(SPEC_CASES))
def test_spectral_loss_per_frame(case, tc, built_lib):
    cfg, B, T = SPEC_CASES[case]
    x, y = _pair(B, T, 30 + T % 97)
    L, taps = _run_spec(cfg, x, y, tc)
    # another configuration in between (the cached arena is rebuilt under a new key), then the same again: same bits
    other = SPEC_CASES["stft_w16_short"][0] if case != "stft_w16_short" else dict(windows=[16], n_mels=[4], fmin=[0.0], fmax=[None])
    _spec_module(other)(x.cuda(), y.cuda())
    L2, _ = _run_spec(cfg, x, y, tc)
    assert torch.equal(L, L2), "two calls differ"
    x64, y64 = x.double(), y.double()
    pw, eps = cfg.get("pow", 2.0), cfg.get("eps", 1e-5)
    v_mag, v_log, ulps = [], [], 0.0
    tag = f"spec {case} tc={tc}"
    for i, (w, nb, ld, Fr, nm) in enumerate(_spec_cfg_geom(cfg, T)):
        X, sabs, fbr = _spec_reference(cfg, x64, y64, i, w)
        fb = None
        if nm:
            fb = taps[f"spec.fb.{i}"].view(nb, nm).double()
            _check_fb(f"{tag} w={w} fb", fb, *fbr)
        c = _dft_coef(w, tc == 2)
        _, re, im = _check_dft(f"{tag} w={w} dft", taps[f"spec.dft.{i}"], X, sabs, c, B, Fr, nb, ld)
        tr = taps[f"spec.terms.{i}"].view(B * Fr, 2).double()
        t1, e1, t2, e2 = _spec_terms(re, im, torch.zeros(2 * B * Fr, dtype=torch.float64), fb, B, Fr, eps, pw)
        _check(f"{tag} w={w} terms.mag", (tr[:, 0] - t1).abs(), e1)
        _check(f"{tag} w={w} terms.log", (tr[:, 1] - t2).abs(), e2)
        t1c, e1c, t2c, e2c = _spec_terms(X.real, X.imag, c * sabs, fb, B, Fr, eps, pw)
        _check(f"{tag} w={w} chain.mag", (tr[:, 0] - t1c).abs(), e1c)
        _check(f"{tag} w={w} chain.log", (tr[:, 1] - t2c).abs(), e2c)
        n_out = nm or nb
        v_mag.append(float(tr[:, 0].sum()) / (B * Fr * n_out))
        v_log.append(float(tr[:, 1].sum()) / (B * Fr * n_out))
        ulps += abs(cfg.get("mw", 1.0)) * _ulp32(v_mag[-1]) + abs(cfg.get("lw", 1.0)) * _ulp32(v_log[-1])
    rec = _spec_combine(v_mag, v_log, cfg.get("mw", 1.0), cfg.get("lw", 1.0))
    # the kernel's fp64 sums round to fp32 on their own: each may land 1 ulp away from ours, then 2 ulps of the combine
    _check(f"{tag} loss", torch.tensor([abs(float(L) - float(rec))]), torch.tensor([ulps + 2 * _ulp32(rec)]))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 262143, 262145, 3 * 1024 * 256 + 17])
def test_l1_and_mse_partials(n, built_lib):
    """absdiff_partial / sqdiff_partial over 1024 blocks of 256 threads (n beyond 1024 x 256 loops the grid), then
    strided_sum: within the float-partials bound 2u of the fp64 mean."""
    from facodec_b200 import losses
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, generator=g)
    y = x * 0.5 + 0.1 * torch.randn(n, generator=g)
    l1 = losses.L1Loss()
    got = [l1(x.cuda(), y.cuda()), l1(x.cuda(), y.cuda())]
    torch.cuda.synchronize()
    assert torch.equal(got[0], got[1])
    ref = float((x.double() - y.double()).abs().mean())
    _check(f"l1 n={n}", torch.tensor([abs(float(got[0]) - ref)]), torch.tensor([2 * U * ref * (1 + 1e-9)]))
    if n > 1024:                                         # the mse term of the reconstruction loss (T > 1024)
        _, terms = losses.reconstruction_loss(x[None].cuda(), y[None].cuda(), return_terms=True)
        mse = float(((x.double() - y.double()) ** 2).mean())
        _check(f"mse n={n}", torch.tensor([abs(float(terms[0]) - mse)]), torch.tensor([2 * U * mse * (1 + 1e-9)]))


# ---------------------------------------------------------------------------------------------------------------------
# mutations: the bounds see subtly wrong references
# ---------------------------------------------------------------------------------------------------------------------
def _recon_components(re, im, fb, B, Fr, eps=EPS_RECON, drop_last=False):
    """(l1, l2) of one reconstruction scale in fp64 from DFT rows (the mutants' values)."""
    t1, _, t2, _ = _recon_terms(re, im, torch.zeros(re.shape[0], dtype=torch.float64), fb, B, Fr, eps)
    if drop_last:
        keep = torch.ones(B * Fr, dtype=torch.bool)
        keep[Fr - 1::Fr] = False
        t1, t2 = t1[keep], t2[keep]
    return float(t1.sum()) / (t1.numel() * 64.0), float(t2.sum()) / t2.numel()


def _shift1(w):
    return torch.cat([w[:, 1:], w[:, -1:]], 1)


def _mutants_recon(x64, g64, s_idx, fb64):
    s, n_fft, nb, ld = _recon_geom(s_idx)
    w2 = torch.cat([x64, g64])
    fb_band = fb64.clone()
    fb_band[:, 30] = torch.roll(fb64[:, 30], 1)
    X = _stft64(w2, n_fft, s)
    Fr = X.shape[0] // w2.shape[0]
    edge = X.clone()
    edge[0::Fr] *= 1.02
    edge[Fr - 1::Fr] *= 1.02
    return {
        "edge_frames_2pct": dict(X=edge),
        "shift_one_sample": dict(X=_stft64(_shift1(w2), n_fft, s)),
        "zero_padding": dict(X=_stft64(w2, n_fft, s, pad_mode="constant")),
        "replicate_padding": dict(X=_stft64(w2, n_fft, s, pad_mode="replicate")),
        "symmetric_hann": dict(X=_stft64(w2, n_fft, s, window=_hann(s, periodic=False))),
        "last_frame_dropped": dict(drop_last=True),
        "band_shifted": dict(fb=fb_band),
        "eps_1e-5": dict(eps=1e-5),
    }


def mutant_scalar_misses(x64, g64, s_idx=0):
    """{mutation: whether |reference - mutant| <= SCALAR_REL |mutant| on both components of scale s_idx} (fp64, CPU)."""
    s, n_fft, nb, ld = _recon_geom(s_idx)
    B, T = x64.shape
    Fr = T // (s // 4) + 1
    w2 = torch.cat([x64, g64])
    X = _stft64(w2, n_fft, s)
    fb64 = _htk_fb64(nb)[0]
    ref = _recon_components(X.real, X.imag, fb64, B, Fr)
    out = {}
    for name, m in _mutants_recon(x64, g64, s_idx, fb64).items():
        Xm = m.get("X", X)
        mut = _recon_components(Xm.real, Xm.imag, m.get("fb", fb64), B, Fr, m.get("eps", EPS_RECON), m.get("drop_last", False))
        out[name] = all(abs(a - b) <= SCALAR_REL * abs(b) for a, b in zip(ref, mut))
    return out


SCALAR_MISSES = {"edge_frames_2pct"}


@pytest.mark.gpu
def test_mutants_are_seen(built_lib):
    """Every mutant reference differs from the kernel by more than the elementwise bound somewhere; the scalar
    tolerance misses exactly SCALAR_MISSES at the benchmark shape (scale s = 64)."""
    x, g = _pair(4, 96000, 5)
    B, T = x.shape
    x64, g64 = x.double(), g.double()
    L, terms, taps = _run_recon(x, g, 2)
    s, n_fft, nb, ld = _recon_geom(0)
    Fr = T // (s // 4) + 1
    fb = taps["recon.fb.0"].view(nb, 64).double()
    tr = taps["recon.terms.0"].view(B * Fr, 2).double()
    re, im, _ = _split_rows(taps["recon.dft.0"], 2 * B * Fr, ld, nb)
    w2 = torch.cat([x64, g64])
    sabs = _sabs(w2, s)
    c = _dft_coef(s, True)
    fb64, bp, norm, freqs = _htk_fb64(nb)
    zero_e = torch.zeros(2 * B * Fr, dtype=torch.float64)
    seen = {}
    for name, m in _mutants_recon(x64, g64, 0, fb64).items():
        if "X" in m:                                    # DFT rows against the mutant
            err = torch.maximum((re - m["X"].real).abs(), (im - m["X"].imag).abs())
            seen[name] = bool((err > (c * sabs)[:, None]).any())
        elif "fb" in m:                                 # the filterbank and the frame terms against the mutant
            fbe = (fb - m["fb"]).abs() > _fb_bound(m["fb"], bp, norm, freqs)[0]
            t1, e1, _, _ = _recon_terms(re, im, zero_e, m["fb"], B, Fr)
            seen[name] = bool(fbe.any()) and bool(((tr[:, 0] - t1).abs() > e1).any())
        elif m.get("drop_last"):                        # the component against the mutant's mean over F - 1 frames
            l1m, _ = _recon_components(re, im, fb, B, Fr, drop_last=True)
            seen[name] = abs(float(terms[1]) - l1m) > _ulp32(l1m)
        else:                                           # eps: the frame terms against the mutant's
            _, _, t2, e2 = _recon_terms(re, im, zero_e, fb, B, Fr, eps=m["eps"])
            seen[name] = bool(((tr[:, 1] - t2).abs() > e2).any())
    # pow ignored, on the spectral loss: the kernel's log terms against pow = 1
    cfg = dict(windows=[512], pow=2.0)
    Ls, staps = _run_spec(cfg, x[:1, :24000], g[:1, :24000], 2)
    nb5, ld5 = _spec_geom(512)
    F5 = 24000 // 128 + 1
    re5, im5, _ = _split_rows(staps["spec.dft.0"], 2 * F5, ld5, nb5)
    _, _, t2, e2 = _spec_terms(re5, im5, torch.zeros(2 * F5, dtype=torch.float64), None, 1, F5, 1e-5, 1.0)
    seen["pow_ignored"] = bool(((staps["spec.terms.0"].view(F5, 2)[:, 1].double() - t2).abs() > e2).any())
    print("MUTANTS seen:", seen)
    assert all(seen.values()), seen
    # the scalar test's view of the same mutants (eps on a signal with silent stretches, where it matters)
    misses = mutant_scalar_misses(x64, g64)
    xs, gs = _silent_pair()
    misses["eps_1e-5"] = mutant_scalar_misses(xs.double(), gs.double())["eps_1e-5"]
    print("MUTANTS missed by the scalar tolerance:", sorted(k for k, v in misses.items() if v))
    assert {k for k, v in misses.items() if v} == SCALAR_MISSES


# ---------------------------------------------------------------------------------------------------------------------
# CPU only: the references themselves
# ---------------------------------------------------------------------------------------------------------------------
def _recon_loss64(x64, g64):
    B, T = x64.shape
    comps = [float(((x64 - g64) ** 2).mean())]
    for i in range(6):
        s, n_fft, nb, ld = _recon_geom(i)
        Fr = T // (s // 4) + 1
        X = _stft64(torch.cat([x64, g64]), n_fft, s)
        comps += list(_recon_components(X.real, X.imag, _htk_fb64(nb)[0], B, Fr))
    L = 100 * comps[0] + sum(comps[1 + 2 * i] + math.sqrt((64 << i) / 2) * comps[2 + 2 * i] for i in range(6))
    return L, comps


def _spec_loss64(cfg, x64, y64):
    B, T = x64.shape
    L = 0.0
    for i, (w, nb, ld, Fr, nm) in enumerate(_spec_cfg_geom(cfg, T)):
        X, _, fbr = _spec_reference(cfg, x64, y64, i, w)
        t1, _, t2, _ = _spec_terms(X.real, X.imag, torch.zeros(X.shape[0], dtype=torch.float64), fbr[0] if fbr else None,
                                   B, Fr, cfg.get("eps", 1e-5), cfg.get("pow", 2.0))
        n = B * Fr * (nm or nb)
        L += cfg.get("lw", 1.0) * float(t2.sum()) / n + cfg.get("mw", 1.0) * float(t1.sum()) / n
    return L


def test_references_match_golden_and_oracle():
    """The fp64 references of this file, reduced to the loss values, against tests/golden/recon_loss.npz (the imported
    reference's fp32 values) and the oracle's fp32 restatements, within fp32 tolerance."""
    import os
    from conftest import ROOT
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    gold = np.load(os.path.join(ROOT, "tests", "golden", "recon_loss.npz"))
    x, g = synth.synth_loss_pair(int(gold["B"]), int(gold["T"]), int(gold["seed"]))
    L, comps = _recon_loss64(x[:, 0].double(), g[:, 0].double())
    assert abs(L - float(gold["loss"])) <= 1e-5 * abs(float(gold["loss"]))
    assert np.all(np.abs(np.array(comps) - gold["terms"]) <= 1e-5 * np.abs(gold["terms"])), (comps, gold["terms"])
    x, g = _pair(2, 5001, 9)
    with torch.no_grad():
        Lo, to = O.reconstruction_loss(x, g, return_terms=True)
    L, comps = _recon_loss64(x.double(), g.double())
    assert abs(L - float(Lo)) <= 1e-5 * abs(float(Lo))
    assert np.all(np.abs(np.array(comps) - to.double().numpy()) <= 1e-5 * to.double().abs().numpy())
    for name in ("stft_all_windows", "mel_44k", "mel_16k", "mel_train"):
        cfg, B, T = SPEC_CASES[name]
        x, y = _pair(B, max(T, 4097), 40)
        kw = dict(window_lengths=cfg["windows"], clamp_eps=cfg.get("eps", 1e-5), mag_weight=cfg.get("mw", 1.0),
                  log_weight=cfg.get("lw", 1.0), pow=cfg.get("pow", 2.0))
        with torch.no_grad():
            if cfg.get("n_mels"):
                ref = O.mel_spectrogram_loss(x[:, None], y[:, None], cfg.get("sr", 24000), n_mels=cfg["n_mels"], mel_fmin=cfg["fmin"],
                                             mel_fmax=cfg["fmax"], **kw)
            else:
                ref = O.multiscale_stft_loss(x[:, None], y[:, None], **kw)
        got = _spec_loss64(cfg, x.double(), y.double())
        assert abs(got - float(ref)) <= 2e-5 * abs(float(ref)), (name, got, float(ref))


def test_scalar_misses_claim_cpu():
    """The docstring's list of mutants the scalar tolerance would miss, from the fp64 references alone."""
    x, g = _pair(4, 96000, 5)
    misses = mutant_scalar_misses(x.double(), g.double())
    xs, gs = _silent_pair()
    misses["eps_1e-5"] = mutant_scalar_misses(xs.double(), gs.double())["eps_1e-5"]
    assert {k for k, v in misses.items() if v} == SCALAR_MISSES, misses
