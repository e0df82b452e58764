"""Training-side losses of the reference on the front-end kernels: ``reconstruction_loss`` (losses.py:65-89, forward value
only) and the ``dac/nn/loss.py`` criteria train.py:153-164 builds (``MultiScaleSTFTLoss``, ``MelSpectrogramLoss``, ``L1Loss``;
their audiotools / librosa arithmetic is restated from the published semantics -- parity unpinned, see the classes), which
back-propagate through torch autograd into both of their inputs.

``reconstruction_loss(x, G_x)`` mirrors losses.py:65-89: ``100 * mse(x, G_x)`` plus, for s = 64 ... 2048, ``l1 + sqrt(s/2) * l2``
between 64-band torchaudio mel spectrograms (``sample_rate=16000, n_fft=max(s,512), win_length=s, hop_length=s//4``).  Per
scale the two signals' frames go through ONE tensor-core GEMM against the window-folded DFT basis, a per-frame kernel
forms both mel spectra and the frame's share of the two terms, and fp64 sums in a fixed order give the scalars
(``fac_reconstruction_loss``).  Forward only -- no autograd graph is attached to the result (SURVEY.md 8f rank 3 stops
at the loss value); a CPU tensor or a missing library raises ``FacError``.

Gradients of the criteria: each loss L is a scalar, so dL/dx * g is exact for any upstream g.  When an input requires grad,
the forward call itself computes dL/dx and / or dL/dy for g = 1 (``fac_spectral_loss_grad`` / ``fac_l1_loss_grad``: per scale a
gradient kernel over the spectra, the transposed DFT GEMM and a deterministic overlap-add) and keeps only those [B, T]
tensors; backward is ``grad_output * saved`` on the device (no saved spectra, no host sync).  The loss value is the one
the no-grad call returns, bit for bit; gradients are bit-reproducible.  Double backward is not supported.
"""
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .modules import Engine, _ptr, _stream

LAMBDA_WAV = 100            # losses.py:58

_ENGINE = None


def _engine(device):
    global _ENGINE
    if _ENGINE is None:
        _ENGINE = Engine()
    _ENGINE._ensure(device)
    return _ENGINE


def _flat(t, name):
    if not torch.is_tensor(t) or t.device.type != "cuda":
        raise _lib.FacError(f"reconstruction_loss: {name} must be a CUDA tensor (there is no CPU path)")
    if t.dim() == 3 and t.shape[1] == 1:
        t = t[:, 0]
    if t.dim() == 1:
        t = t[None]
    if t.dim() != 2:
        raise _lib.FacError(f"reconstruction_loss: {name} must be [B, T] or [B, 1, T], got {tuple(t.shape)}")
    return t.float().contiguous()


def reconstruction_loss(x, G_x, eps=1e-7, return_terms=False):
    """losses.py:65-89.  x, G_x: [B, 1, T] or [B, T] on the GPU, T > 1024.  Returns the 0-d loss (and, with
    ``return_terms``, the 13 components: mse, then (l1, l2) for s = 64, 128, ..., 2048).

    Forward only: the result carries no autograd graph (train.py does not use this loss).  Its l2 term,
    sqrt(mean over bands of the squared log-mel difference), has no derivative where a frame's difference is zero, and
    torch autograd of the reference gives NaN there."""
    if eps != 1e-7:
        raise _lib.FacError("reconstruction_loss: eps is fixed at the reference's 1e-7")
    a, b = _flat(x, "x"), _flat(G_x, "G_x")
    if a.shape != b.shape or a.device != b.device:
        raise _lib.FacError(f"reconstruction_loss: shapes / devices differ: {tuple(a.shape)} vs {tuple(b.shape)}")
    e = _engine(a.device)
    out = torch.empty(14, device=a.device)
    B, T = a.shape
    _lib.check(e.handle, e.L.fac_reconstruction_loss(e.handle, _ptr(a), _ptr(b), B, T, _ptr(out), _ptr(out[1:]), _stream(a.device)),
               "fac_reconstruction_loss")
    return (out[0], out[1:]) if return_terms else out[0]


# ---- dac/nn/loss.py:11-47, :142-327 ------------------------------------------------------------------------------------
def _signal(x, name):
    """A [B, T] / [B, 1, T] CUDA tensor, or an AudioSignal-like object (``.audio_data``, ``.sample_rate``)."""
    sr = getattr(x, "sample_rate", None)
    t = getattr(x, "audio_data", x)
    return _flat(t, name), sr


class _LossWithGrad(torch.autograd.Function):
    """``run(a, b, want_a, want_b) -> (loss, dL/da or None, dL/db or None)``, one device call; backward scales the saved
    gradients by the upstream one."""

    @staticmethod
    def forward(ctx, run, a, b):
        loss, da, db = run(a, b, ctx.needs_input_grad[1], ctx.needs_input_grad[2])
        ctx.save_for_backward(da, db)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        da, db = ctx.saved_tensors
        return None, (g * da if da is not None else None), (g * db if db is not None else None)


def _apply(run, a, b):
    if torch.is_grad_enabled() and (a.requires_grad or b.requires_grad):
        return _LossWithGrad.apply(run, a, b)
    return run(a, b, False, False)[0]


class _Criterion:
    def to(self, *args, **kwargs):
        """The criteria hold no tensors (their constants live on the device the inputs come from): returns self, so
        ``criterion.to(device)`` as train.py:154-164 writes it keeps working."""
        return self


class L1Loss(_Criterion):
    """dac/nn/loss.py:11-47 L1Loss(attribute='audio_data'): mean |x - y| (``weight`` is stored, not applied, as in the reference).
    Differentiable in both inputs: dL/dx = sgn(x - y) / n (0 where x == y, as torch), dL/dy = -dL/dx."""

    def __init__(self, attribute="audio_data", weight=1.0):
        if attribute != "audio_data":
            raise NotImplementedError("only the waveform attribute is built")
        self.attribute, self.weight = attribute, weight

    def __call__(self, x, y):
        a, _ = _signal(x, "x")
        b, _ = _signal(y, "y")
        if a.shape != b.shape or a.device != b.device:
            raise _lib.FacError(f"L1Loss: shapes / devices differ: {tuple(a.shape)} vs {tuple(b.shape)}")

        def run(a, b, want_a, want_b):
            e = _engine(a.device)
            if not (want_a or want_b):
                out = torch.empty(1, device=a.device)
                _lib.check(e.handle, e.L.fac_l1_loss(e.handle, _ptr(a), _ptr(b), a.numel(), _ptr(out), _stream(a.device)), "fac_l1_loss")
                return out[0], None, None
            out = torch.empty((), device=a.device)
            da = torch.empty_like(a) if want_a else None
            db = torch.empty_like(b) if want_b else None
            _lib.check(e.handle, e.L.fac_l1_loss_grad(e.handle, _ptr(a), _ptr(b), a.numel(), _ptr(out), _ptr(da), _ptr(db),
                                                       _stream(a.device)), "fac_l1_loss_grad")
            return out, da, db

        return _apply(run, a, b)

    forward = __call__


class _SpectralLoss(_Criterion):
    def _run(self, x, y, n_mels, fmin, fmax):
        import ctypes
        a, sra = _signal(x, "x")
        b, _ = _signal(y, "y")
        if a.shape != b.shape or a.device != b.device:
            raise _lib.FacError(f"{type(self).__name__}: shapes / devices differ: {tuple(a.shape)} vs {tuple(b.shape)}")
        sr = int(sra if sra is not None else self.sample_rate)
        n = len(self.window_lengths)
        wl = (ctypes.c_int * n)(*self.window_lengths)
        nm = (ctypes.c_int * n)(*n_mels) if n_mels is not None else None
        f0 = (ctypes.c_float * n)(*[float(v) for v in fmin]) if n_mels is not None else None
        f1 = (ctypes.c_float * n)(*[0.0 if v is None else float(v) for v in fmax]) if n_mels is not None else None
        f0p = ctypes.cast(f0, ctypes.c_void_p) if f0 is not None else None
        f1p = ctypes.cast(f1, ctypes.c_void_p) if f1 is not None else None
        consts = (float(self.clamp_eps), float(self.mag_weight), float(self.log_weight), float(self.pow))

        def run(a, b, want_a, want_b):
            e = _engine(a.device)
            B, T = a.shape
            if not (want_a or want_b):
                out = torch.empty(1, device=a.device)
                rc = e.L.fac_spectral_loss(e.handle, _ptr(a), _ptr(b), B, T, sr, n, wl, nm, f0p, f1p, *consts, _ptr(out), _stream(a.device))
                _lib.check(e.handle, rc, "fac_spectral_loss")
                return out[0], None, None
            out = torch.empty((), device=a.device)
            da = torch.empty_like(a) if want_a else None
            db = torch.empty_like(b) if want_b else None
            rc = e.L.fac_spectral_loss_grad(e.handle, _ptr(a), _ptr(b), B, T, sr, n, wl, nm, f0p, f1p, *consts, _ptr(out), _ptr(da),
                                            _ptr(db), _stream(a.device))
            _lib.check(e.handle, rc, "fac_spectral_loss_grad")
            return out, da, db

        return _apply(run, a, b)


class MultiScaleSTFTLoss(_SpectralLoss):
    """dac/nn/loss.py:142-231 (train.py:154 uses the defaults): sum over window lengths of
    ``log_weight * L1(log10(clamp(|X|, eps)^pow), ...) + mag_weight * L1(|X|, |Y|)`` with X = AudioSignal.stft(w, w // 4) --
    restated as torch.stft(periodic Hann, centre = True, reflect); audiotools is not vendored (SURVEY.md 8c): parity
    unpinned.  ``match_stride`` / ``window_type`` other than the defaults and custom ``loss_fn`` are not built.
    Differentiable in both inputs (module docstring)."""

    def __init__(self, window_lengths=(2048, 512), loss_fn=None, clamp_eps=1e-5, mag_weight=1.0, log_weight=1.0, pow=2.0, weight=1.0,
                 match_stride=False, window_type=None, sample_rate=24000):
        if loss_fn is not None or match_stride or window_type not in (None, "hann"):
            raise NotImplementedError("only nn.L1Loss, match_stride=False and the Hann window are built")
        self.window_lengths = [int(w) for w in window_lengths]
        self.clamp_eps, self.mag_weight, self.log_weight, self.pow, self.weight = clamp_eps, mag_weight, log_weight, pow, weight
        self.sample_rate = sample_rate

    def __call__(self, x, y):
        return self._run(x, y, None, None, None)

    forward = __call__


class MelSpectrogramLoss(_SpectralLoss):
    """dac/nn/loss.py:234-327 (train.py:155-163: n_mels 5..320 over windows 32..2048, pow = 1, mag_weight = 0): as above on
    ``AudioSignal.mel_spectrogram`` = |stft| @ librosa.filters.mel(sample_rate, n_fft, n_mels, fmin, fmax).T (Slaney scale and
    area normalisation; restated, cross-checked against torchaudio's Slaney filterbank in tests/test_oracle.py).
    Differentiable in both inputs (module docstring): ``mel_criterion(recons, signal)`` back-propagates into the waveform
    behind ``recons.audio_data``."""

    def __init__(self, n_mels=(150, 80), window_lengths=(2048, 512), loss_fn=None, clamp_eps=1e-5, mag_weight=1.0, log_weight=1.0,
                 pow=2.0, weight=1.0, match_stride=False, mel_fmin=(0.0, 0.0), mel_fmax=(None, None), window_type=None,
                 sample_rate=24000):
        if loss_fn is not None or match_stride or window_type not in (None, "hann"):
            raise NotImplementedError("only nn.L1Loss, match_stride=False and the Hann window are built")
        self.window_lengths = [int(w) for w in window_lengths]
        self.n_mels, self.mel_fmin, self.mel_fmax = [int(v) for v in n_mels], list(mel_fmin), list(mel_fmax)
        if not (len(self.n_mels) == len(self.window_lengths) == len(self.mel_fmin) == len(self.mel_fmax)):
            raise ValueError("n_mels, window_lengths, mel_fmin and mel_fmax must have one entry per scale")
        self.clamp_eps, self.mag_weight, self.log_weight, self.pow, self.weight = clamp_eps, mag_weight, log_weight, pow, weight
        self.sample_rate = sample_rate

    def __call__(self, x, y):
        return self._run(x, y, self.n_mels, self.mel_fmin, self.mel_fmax)

    forward = __call__
