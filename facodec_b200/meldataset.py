"""Dataset-side mel of the reference's training input pipeline (meldataset.py:29-71), computed by the front-end
kernels (frame gather + tensor-core DFT + mel filterbank) through ``fac_dataset_mel``.

``preprocess(wave)`` mirrors meldataset.py:42-47: torchaudio ``MelSpectrogram(n_mels=80, n_fft=2048, win_length=1200,
hop_length=300)`` with its DEFAULT ``sample_rate=16000`` filterbank (not the quantizer's 24 kHz one), then
``(log(1e-5 + mel) + 4) / 4``; returns ``[1, 80, T // 300 + 1]``.  ``PseudoDataset`` is the reference's synthetic
dataset (:50-71).  There is no CPU fallback: the mel is computed on ``device`` (default cuda:0) and returned there.
"""
import ctypes
import random

import numpy as np
import torch

from . import _lib
from .modules import Engine, _ptr, _stream

np.random.seed(114514)      # meldataset.py:26-27
random.seed(114514)
SPECT_PARAMS = {"n_fft": 2048, "win_length": 1200, "hop_length": 300}
MEL_PARAMS = {"n_mels": 80}
mean, std = -4, 4

_ENGINE = None


def _engine(device):
    global _ENGINE
    if _ENGINE is None:
        _ENGINE = Engine()
    _ENGINE._ensure(device)
    return _ENGINE


def to_mel_batch(waves, device=None):
    """waves [B, T] (numpy or tensor) -> normalised log-mel [B, 80, T // 300 + 1] on the GPU."""
    w = torch.from_numpy(waves).float() if isinstance(waves, np.ndarray) else waves.float()
    if w.device.type != "cuda":
        w = w.to(device or torch.device("cuda", torch.cuda.current_device()))
    w = w.contiguous()
    B, T = w.shape
    e = _engine(w.device)
    mel = torch.empty(B, MEL_PARAMS["n_mels"], T // SPECT_PARAMS["hop_length"] + 1, device=w.device)
    _lib.check(e.handle, e.L.fac_dataset_mel(e.handle, _ptr(w), B, T, _ptr(mel), _stream(w.device)), "fac_dataset_mel")
    return mel


def preprocess(wave, device=None):
    """meldataset.py:42-47: wave [T] -> [1, 80, T // 300 + 1]."""
    w = torch.from_numpy(wave).float() if isinstance(wave, np.ndarray) else wave.float()
    return to_mel_batch(w.reshape(1, -1), device)


class PseudoDataset(torch.utils.data.Dataset):
    """meldataset.py:50-71: random-length (1-30 s) Gaussian waves normalised to unit peak, with their mel."""

    def __init__(self, sr=24000, range=(1, 30)):
        self.data_list = []
        self.sr = sr
        self.duration_range = range

    def __len__(self):
        return 100

    def __getitem__(self, idx):
        wave = np.random.randn(self.sr * random.randint(*self.duration_range))
        wave = wave / np.max(np.abs(wave))
        mel = preprocess(wave).squeeze(0)
        wave = torch.from_numpy(wave).float()
        return wave, mel
