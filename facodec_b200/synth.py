"""Deterministic synthetic checkpoints and waveforms for FAcodec (no network => no
trained checkpoint; SURVEY.md section 8c/8d).

``synth_state_dicts(seed)`` returns ``{'encoder': sd, 'quantizer': sd, 'decoder': sd}``
with exactly the key names / shapes / dtypes of the reference checkpoints
(``reconstruct.py:30-34`` loads ``ckpt[key]`` per module; keys listed in
the reference state_dicts).  Values are drawn from ``numpy.random.RandomState`` so
that the same seed gives bit-identical tensors on any machine, following the
default PyTorch initialisers of each layer family so activations have
reference-like statistics:

* Conv1d / ConvTranspose1d / Linear: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias
  (``weight_v``); ``weight_g = ||weight_v||_{dims != 0} * U(0.8, 1.2)`` so the weight-norm
  fold is exercised with g != ||v|| as in a trained model.
* Snake alpha: U(0.5, 1.5) (reference initialises to 1; trained values differ).
* LSTM: U(-1/sqrt(H), 1/sqrt(H)); nn.Embedding codebooks: N(0, 1).
* MultiHeadAttention q/k/v: xavier-uniform (modules/attentions.py:149-153); conv_k is NOT
  tied to conv_q (the reference ties them only at init, :154-157; trained values differ and a
  q/k swap bug must be visible).
* timbre_linear.bias = [1]*1024 + [0]*1024 (modules/quantize.py:196-198) plus small noise.
* ``to_mel.spectrogram.window`` = periodic Hann(1200); ``to_mel.mel_scale.fb`` = HTK
  mel filterbank [1025, 80] for sample_rate 24000, f in [0, 12000], norm=None
  (torchaudio.transforms.MelSpectrogram defaults; modules/quantize.py:228-230).

``synth_waves`` follows meldataset.py:67-68 (PseudoDataset) with fixed length.
"""
import math
from collections import OrderedDict

import numpy as np
import torch

ENC_DIM = 64
ENC_RATES = (2, 5, 5, 6)
DEC_DIM = 1536
DEC_RATES = (6, 5, 5, 2)
LATENT = 1024
HOP = 300
SR = 24000


class _Gen:
    def __init__(self, seed):
        self.rs = np.random.RandomState(seed)

    def uniform(self, shape, bound):
        return torch.from_numpy(self.rs.uniform(-bound, bound, size=shape).astype(np.float32))

    def normal(self, shape):
        return torch.from_numpy(self.rs.standard_normal(size=shape).astype(np.float32))

    def scale(self, shape, lo, hi):
        return torch.from_numpy(self.rs.uniform(lo, hi, size=shape).astype(np.float32))


def _conv(g, sd, prefix, cout, cin, k, weight_norm=True, transposed=False):
    """nn.Conv1d weight [cout, cin, k]; nn.ConvTranspose1d weight [cin, cout, k]
    (weight-norm dim 0 == in-channels there, SURVEY.md 8a7)."""
    shape = (cin, cout, k) if transposed else (cout, cin, k)
    # torch's fan_in is size(1) * receptive field for both layouts
    fan_in = shape[1] * k
    bound = 1.0 / math.sqrt(fan_in)
    v = g.uniform(shape, bound)
    b = g.uniform((cout,), bound)
    if weight_norm:
        # fp64 numpy norm then round: identical bits on every host CPU
        n = np.sqrt((v.numpy().astype(np.float64).reshape(shape[0], -1) ** 2).sum(axis=1))
        n = torch.from_numpy(n.astype(np.float32)).reshape(shape[0], 1, 1)
        sd[prefix + ".bias"] = b
        sd[prefix + ".weight_g"] = n * g.scale((shape[0], 1, 1), 0.8, 1.2)
        sd[prefix + ".weight_v"] = v
    else:
        sd[prefix + ".weight"] = v
        sd[prefix + ".bias"] = b


def _snake(g, sd, name, c):
    sd[name] = g.scale((1, c, 1), 0.5, 1.5)


def _res_unit(g, sd, prefix, c):
    _snake(g, sd, prefix + ".block.0.alpha", c)
    _conv(g, sd, prefix + ".block.1.conv.conv", c, c, 7)
    _snake(g, sd, prefix + ".block.2.alpha", c)
    _conv(g, sd, prefix + ".block.3.conv.conv", c, c, 1)


def _lstm(g, sd, prefix, h, layers=2):
    bound = 1.0 / math.sqrt(h)
    for l in range(layers):
        sd[f"{prefix}.weight_ih_l{l}"] = g.uniform((4 * h, h), bound)
        sd[f"{prefix}.weight_hh_l{l}"] = g.uniform((4 * h, h), bound)
        sd[f"{prefix}.bias_ih_l{l}"] = g.uniform((4 * h,), bound)
        sd[f"{prefix}.bias_hh_l{l}"] = g.uniform((4 * h,), bound)


def synth_encoder(seed):
    """Keys of dac/model/dac.py:69-104 Encoder(d_model=64, strides=[2,5,5,6], d_latent=1024, lstm=2)."""
    g = _Gen(seed)
    sd = {}
    _conv(g, sd, "block.0.conv.conv", ENC_DIM, 1, 7)
    c = ENC_DIM
    for i, s in enumerate(ENC_RATES):
        p = f"block.{i + 1}"
        for j in range(3):
            _res_unit(g, sd, f"{p}.block.{j}", c)
        _snake(g, sd, f"{p}.block.3.alpha", c)
        _conv(g, sd, f"{p}.block.4.conv.conv", 2 * c, c, 2 * s)
        c *= 2
    _lstm(g, sd, "block.5.lstm", c)
    _snake(g, sd, "block.6.alpha", c)
    _conv(g, sd, "block.7.conv.conv", LATENT, c, 3)
    return sd


def synth_decoder(seed, lstm=2):
    """Keys of dac/model/dac.py:131-165 Decoder(1024, 1536, [6,5,5,2], lstm=2); lstm=0 (the redecoder's decoder,
    configs/config_redecoder.yml) drops the SLSTM and shifts the nn.Sequential indices down by one."""
    g = _Gen(seed)
    sd = {}
    _conv(g, sd, "model.0.conv.conv", DEC_DIM, LATENT, 7)
    base = 1
    if lstm:
        _lstm(g, sd, "model.1.lstm", DEC_DIM, layers=lstm)
        base = 2
    c = DEC_DIM
    for i, s in enumerate(DEC_RATES):
        p = f"model.{i + base}"
        _snake(g, sd, f"{p}.block.0.alpha", c)
        _conv(g, sd, f"{p}.block.1.convtr.convtr", c // 2, c, 2 * s, transposed=True)
        for j in range(3):
            _res_unit(g, sd, f"{p}.block.{j + 2}", c // 2)
        c //= 2
    _snake(g, sd, f"model.{4 + base}.alpha", c)
    _conv(g, sd, f"model.{5 + base}.conv.conv", 1, c, 7)
    return sd


def synth_redecoder(seed, embed_dim=512, n_layers=16, gin=1024):
    """Keys of modules/redecoder.py:5-21 Redecoder(encoder_type='wavenet'): WN(hidden 512, kernel 5, 16 layers,
    gin_channels 1024) as ``encoder.*`` (modules/wavenet.py:103-136), conv_out Conv1d(512, 1024, 1), one prosody and two
    content nn.Embedding(1024, 512) (N(0, 1) init)."""
    g = _Gen(seed)
    sd = {}
    _conv(g, sd, "encoder.cond_layer.conv.conv", 2 * embed_dim * n_layers, gin, 1)
    for i in range(n_layers):
        _conv(g, sd, f"encoder.in_layers.{i}.conv.conv", 2 * embed_dim, embed_dim, 5)
    for i in range(n_layers):
        _conv(g, sd, f"encoder.res_skip_layers.{i}.conv.conv", 2 * embed_dim if i < n_layers - 1 else embed_dim, embed_dim, 1)
    _conv(g, sd, "conv_out", LATENT, embed_dim, 1, weight_norm=False)
    sd["prosody_embed.0.weight"] = g.normal((1024, embed_dim))
    for i in range(2):
        sd[f"content_embed.{i}.weight"] = g.normal((1024, embed_dim))
    return sd


def synth_redecoder_state_dicts(seed=0):
    """{'encoder': Redecoder, 'decoder': Decoder(causal=False, lstm=0)} as build_model(stage='redecoder') lays them out
    (modules/commons.py:385-412)."""
    return {"encoder": synth_redecoder(seed * 3 + 101), "decoder": synth_decoder(seed * 3 + 102, lstm=0)}


def synth_cnnlstm(seed, indim, outdim, heads):
    """Keys of modules/quantize.py:106-125 CNNLSTM(indim, outdim, head): model.{0,1,2} = ResidualUnit (block.0 / block.2 =
    Activation1d(SnakeBeta) -> ``act.alpha`` / ``act.beta`` (log scale) plus the registered filter buffers, block.1 /
    block.3 = weight-normed Conv1d k7 / k1), model.3 = Activation1d(SnakeBeta), heads.{i} = nn.Linear."""
    g = _Gen(seed)
    sd = {}
    for j in range(3):
        p = f"model.{j}"
        for blk in (0, 2):
            sd[f"{p}.block.{blk}.act.alpha"] = g.uniform((indim,), 0.3)
            sd[f"{p}.block.{blk}.act.beta"] = g.uniform((indim,), 0.3)
        _conv(g, sd, f"{p}.block.1", indim, indim, 7)
        _conv(g, sd, f"{p}.block.3", indim, indim, 1)
    sd["model.3.act.alpha"] = g.uniform((indim,), 0.3)
    sd["model.3.act.beta"] = g.uniform((indim,), 0.3)
    b = 1.0 / math.sqrt(indim)
    for i in range(heads):
        sd[f"heads.{i}.weight"] = g.uniform((outdim, indim), b)
        sd[f"heads.{i}.bias"] = g.uniform((outdim,), b)
    return sd


def hann_window_periodic(n):
    """torch.hann_window(n, periodic=True): 0.5 - 0.5 cos(2 pi i / n), computed in fp64 then
    rounded (within 1 ulp of torch's fp32 evaluation)."""
    i = np.arange(n, dtype=np.float64)
    return torch.from_numpy((0.5 - 0.5 * np.cos(2.0 * np.pi * i / n)).astype(np.float32))


def melscale_fbanks_htk(n_freqs=1025, f_min=0.0, f_max=12000.0, n_mels=80, sample_rate=24000):
    """torchaudio.functional.melscale_fbanks(norm=None, mel_scale='htk') formula, evaluated in
    fp64 numpy and rounded once (host-independent bits; within 1e-6 of torchaudio's fp32
    evaluation, checked in tests/test_host.py)."""
    all_freqs = np.linspace(0, sample_rate // 2, n_freqs)
    m_min = 2595.0 * math.log10(1.0 + (f_min / 700.0))
    m_max = 2595.0 * math.log10(1.0 + (f_max / 700.0))
    m_pts = np.linspace(m_min, m_max, n_mels + 2)
    f_pts = 700.0 * (10 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    fb = np.maximum(0.0, np.minimum(down, up))
    return torch.from_numpy(fb.astype(np.float32))


def _vq(g, sd, prefix, dim=LATENT, cb_dim=8, cb_size=1024):
    _conv(g, sd, prefix + ".in_proj", cb_dim, dim, 1)
    _conv(g, sd, prefix + ".out_proj", dim, cb_dim, 1)
    sd[prefix + ".codebook.weight"] = g.normal((cb_size, cb_dim))


def synth_quantizer(seed):
    """Keys of modules/quantize.py:156-237 FAquantizer(in_dim=1024, n_p=1, n_c=2, n_r=3,
    separate_prosody_encoder=True, timbre_norm=True)."""
    g = _Gen(seed)
    sd = {}
    _vq(g, sd, "prosody_quantizer.quantizers.0")
    for i in range(2):
        _vq(g, sd, f"content_quantizer.quantizers.{i}")
    # StyleEncoder(in_dim=80, hidden_dim=512, out_dim=1024), modules/style_encoder.py:33-61
    _conv(g, sd, "timbre_encoder.spectral.0", 512, 80, 1, weight_norm=False)
    _conv(g, sd, "timbre_encoder.spectral.3", 512, 512, 1, weight_norm=False)
    for i in range(2):
        _conv(g, sd, f"timbre_encoder.temporal.{i}.conv1", 1024, 512, 5, weight_norm=False)
    xb = math.sqrt(6.0 / (512 + 512))
    for n in ("q", "k", "v", "o"):
        _conv(g, sd, f"timbre_encoder.slf_attn.conv_{n}", 512, 512, 1, weight_norm=False)
        if n in ("q", "k", "v"):
            sd[f"timbre_encoder.slf_attn.conv_{n}.weight"] = g.uniform((512, 512, 1), xb)
    _conv(g, sd, "timbre_encoder.fc", 1024, 512, 1, weight_norm=False)
    b = 1.0 / math.sqrt(1024)
    sd["timbre_linear.weight"] = g.uniform((2048, 1024), b)
    tb = torch.cat([torch.ones(1024), torch.zeros(1024)]) + g.uniform((2048,), 0.05)
    sd["timbre_linear.bias"] = tb
    for i in range(3):
        _vq(g, sd, f"residual_quantizer.quantizers.{i}")
    _conv(g, sd, "melspec_linear.conv.conv", 256, 20, 1, weight_norm=False)
    for i in range(8):
        _conv(g, sd, f"melspec_encoder.in_layers.{i}.conv.conv", 512, 256, 5)
    for i in range(8):
        _conv(g, sd, f"melspec_encoder.res_skip_layers.{i}.conv.conv", 512 if i < 7 else 256, 256, 1)
    _conv(g, sd, "melspec_linear2.conv.conv", 1024, 256, 1, weight_norm=False)
    sd["to_mel.spectrogram.window"] = hann_window_periodic(1200)
    sd["to_mel.mel_scale.fb"] = melscale_fbanks_htk()
    return sd


def synth_state_dicts(seed=0):
    return {
        "encoder": synth_encoder(seed * 3 + 1),
        "quantizer": synth_quantizer(seed * 3 + 2),
        "decoder": synth_decoder(seed * 3 + 3),
    }


def synth_loss_pair(batch, n_samples, seed=11):
    """(x, G_x) for the reconstruction-loss fixtures: x = synth_waves, G_x = 0.7 x + 0.05 n (n from a numpy RandomState:
    host-independent bits, exact fp32 arithmetic).  Both float32 [batch, 1, n_samples]."""
    x = synth_waves(batch, n_samples, seed=seed)
    n = np.random.RandomState(seed + 7).randn(batch, 1, n_samples).astype(np.float32)
    g = np.float32(0.7) * x.numpy() + np.float32(0.05) * n
    return x, torch.from_numpy(g.astype(np.float32))


def synth_waves(batch, n_samples=4 * SR, seed=114514):
    """PseudoDataset law (meldataset.py:67-68): randn(n)/max|.|, seed from meldataset.py:26;
    utterance i uses the next n_samples draws. Returns float32 [batch, 1, n_samples]."""
    rs = np.random.RandomState(seed)
    out = np.empty((batch, 1, n_samples), dtype=np.float32)
    for i in range(batch):
        w = rs.randn(n_samples)
        w = w / np.max(np.abs(w))
        out[i, 0] = w.astype(np.float32)
    return torch.from_numpy(out)


def synth_jdc(seed=0):
    """Synthetic weights of JDCNet(num_class=1, seq_len=192) (modules/JDC/model.py) under its state-dict keys: 2-D convs
    and linears at 1/sqrt(fan_in), BatchNorms with non-trivial affine parameters and running statistics, and a classifier
    weight of 40 / sqrt(512) and bias of 4.5, so that F0 = |classifier| falls on both sides of train.py's 5.0 voiced threshold."""
    from .modules import JDCNet
    g = _Gen(700 + seed)
    sd = OrderedDict()
    for k, t in JDCNet().state_dict().items():
        shape = tuple(t.shape)
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(1000, dtype=torch.long)
        elif k.endswith("running_mean"):
            sd[k] = g.uniform(shape, 0.2)
        elif k.endswith("running_var"):
            sd[k] = g.scale(shape, 0.5, 1.5)
        elif len(shape) == 1 and not k.startswith(("bilstm", "classifier", "detector.")):
            sd[k] = g.scale(shape, 0.8, 1.2) if k.endswith("weight") else g.uniform(shape, 0.1)   # BatchNorm affine
        elif k.startswith("bilstm"):
            sd[k] = g.uniform(shape, 1.0 / math.sqrt(256))
        elif k == "classifier.bias":
            sd[k] = torch.full(shape, 4.5)
        else:
            fan_in = int(np.prod(shape[1:])) if len(shape) > 1 else shape[0]
            sd[k] = g.uniform(shape, (40.0 if k == "classifier.weight" else 1.0) / math.sqrt(fan_in))
    return sd
