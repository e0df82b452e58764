"""Reference-facing call surface:  model.encoder(x) / model.quantizer(z, wave, ...) /
model.decoder(z)  on the Munch returned by build_model (reference modules/commons.py:283-348),
backed by the C-ABI library (include/facodec_b200.h).  PyTorch here is plumbing only: it owns
the device tensors and the CUDA stream; all arithmetic happens in libfacodec_b200.so.

Drop-in contract (SURVEY.md section 8b):
* ``Encoder`` / ``FAquantizer`` / ``Decoder`` are nn.Modules whose ``state_dict()`` /
  ``load_state_dict()`` use the reference's key names (legacy weight-norm ``weight_g`` /
  ``weight_v`` included), so reference checkpoints load unchanged (reconstruct.py:30-34).
* forward signatures and returns are those of dac/model/dac.py:103-104, :164-165 and
  modules/quantize.py:375-454 (forward_v2).  Inference only (eval mode, no autograd): the
  training-time branches (quantizer dropout, random residual mask) are out of scope.
* There is no CPU fallback: CPU tensors or a missing library raise.
"""
import ctypes
import json
import math
import operator
import os
import struct
from collections import OrderedDict

import torch
from torch import nn

from . import _lib, synth

MOD_ENCODER, MOD_QUANTIZER, MOD_DECODER, MOD_REDECODER, MOD_REDEC_DECODER = 0, 1, 2, 3, 4


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(device=None):
    """The current CUDA stream OF THE TENSORS' DEVICE (not of whatever device happens to be current)."""
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class Engine:
    """One fac_handle (one CUDA device).  The three modules of a build_model() share it so that
    codec_forward can run encoder -> quantizer -> decoder inside one C call."""

    def __init__(self):
        self.L = _lib.load()
        self.handle = None
        self.device_index = None
        self.loaded_version = {}
        self.modules = {}
        self._rs_pairs = set()      # reduced rate pairs whose resampler table this handle holds

    def _ensure(self, device):
        if device.type != "cuda":
            raise _lib.FacError("facodec_b200 runs on CUDA tensors only (no CPU fallback); got " + str(device))
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if self.handle is None:
            h = ctypes.c_void_p()
            rc = self.L.fac_create(ctypes.byref(h), idx)
            if rc < 0:
                raise _lib.FacError(f"fac_create(device={idx}) failed with status {rc}")
            self.handle, self.device_index = h, idx
            # measurement aid: FACODEC_B200_OPTS="name=value,name=value" applies fac_set_option at creation
            for kv in filter(None, os.environ.get("FACODEC_B200_OPTS", "").split(",")):
                name, _, val = kv.partition("=")
                _lib.check(self.handle, self.L.fac_set_option(self.handle, name.strip().encode(), int(val)), "fac_set_option")
        elif idx != self.device_index:
            raise _lib.FacError("engine is bound to cuda:%d, got cuda:%d" % (self.device_index, idx))

    def set_option(self, name, value, device=None):
        """fac_set_option, e.g. ("tensor_cores", 0|1|2)."""
        self._ensure(device or torch.device("cuda", torch.cuda.current_device()))
        _lib.check(self.handle, self.L.fac_set_option(self.handle, name.encode(), int(value)), "fac_set_option")

    def register(self, module_id, module):
        self.modules[module_id] = module

    def sync_weights(self, device):
        """(Re)uploads the weights of every registered module whose parameters changed."""
        self._ensure(device)
        dirty = [m for m, mod in self.modules.items() if self.loaded_version.get(m) != mod._version_tag()]
        if not dirty:
            return
        # fac_finalize repacks everything it holds, so push all registered modules again
        for m, mod in self.modules.items():
            for key, t in mod.state_dict().items():
                t = t.detach().to("cpu", torch.float32).contiguous()
                shape = (ctypes.c_int64 * max(t.dim(), 1))(*t.shape)
                rc = self.L.fac_load_tensor(self.handle, m, key.encode(), _ptr(t), shape, t.dim())
                _lib.check(self.handle, rc, "fac_load_tensor(%s)" % key)
        _lib.check(self.handle, self.L.fac_finalize(self.handle), "fac_finalize")
        for m, mod in self.modules.items():
            self.loaded_version[m] = mod._version_tag()

    def __del__(self):
        try:
            if self.handle is not None:
                self.L.fac_destroy(self.handle)
        except Exception:
            pass


class _RefKeyModule(nn.Module):
    """nn.Module whose parameters are stored flat but exposed under the reference's dotted keys."""

    _module_id = None
    _buffer_keys = ()

    def __init__(self, init_sd, engine=None, module_id=None):
        super().__init__()
        if module_id is not None:
            self._module_id = module_id
        self._keys = list(init_sd.keys())
        self._p = nn.ParameterDict()
        for k, v in init_sd.items():
            if k in self._buffer_keys:
                self.register_buffer(self._safe(k), v.clone(), persistent=True)
            else:
                self._p[self._safe(k)] = nn.Parameter(v.clone(), requires_grad=False)
        self._load_count = 0
        self._engine = engine if engine is not None else Engine()
        self._engine.register(self._module_id, self)

    @staticmethod
    def _safe(k):
        return k.replace(".", "/")

    def _get(self, k):
        s = self._safe(k)
        return self._p[s] if s in self._p else getattr(self, s)

    def _version_tag(self):
        return (self._load_count,) + tuple(self._get(k)._version for k in self._keys)

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False, **kw):
        out = destination if destination is not None else OrderedDict()
        for k in self._keys:
            t = self._get(k)
            out[prefix + k] = t if keep_vars else t.detach()
        return out

    def load_state_dict(self, state_dict, strict=True, assign=False):
        missing = [k for k in self._keys if k not in state_dict]
        unexpected = [k for k in state_dict if k not in self._keys]
        if strict and (missing or unexpected):
            raise RuntimeError("Error(s) in loading state_dict for %s: missing %s unexpected %s"
                               % (type(self).__name__, missing[:5], unexpected[:5]))
        with torch.no_grad():
            for k in self._keys:
                if k in state_dict:
                    dst = self._get(k)
                    src = state_dict[k]
                    if tuple(src.shape) != tuple(dst.shape):
                        raise RuntimeError("size mismatch for %s: %s vs %s" % (k, tuple(src.shape), tuple(dst.shape)))
                    dst.copy_(src)
        self._load_count += 1
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def _prep(self, *tensors):
        """Every tensor argument must live on the engine's CUDA device: a CPU tensor or one on another GPU would hand the
        kernels a foreign pointer (illegal address, sticky context error) instead of the promised FacError."""
        if self.training:
            raise NotImplementedError("facodec_b200 implements the eval-mode forward only; call .eval()")
        dev = tensors[0].device
        self._engine.sync_weights(dev)
        for t in tensors[1:]:
            if t is None:
                continue
            if t.device.type != "cuda" or (t.device.index if t.device.index is not None else torch.cuda.current_device()) != self._engine.device_index:
                raise _lib.FacError("all inputs must be on cuda:%d (no CPU fallback, no cross-device copies); got %s"
                                    % (self._engine.device_index, t.device))
        return self._engine.L, self._engine.handle


def _f32c(t):
    return t.detach().to(torch.float32).contiguous()


def _engine_inputs(engine, tensors):
    """Uploads the engine's weights to the first tensor's device if they changed, and raises FacError for any tensor that is
    not on the engine's CUDA device (no CPU fallback, no cross-device copies)."""
    engine.sync_weights(tensors[0].device)
    for t in tensors:
        if t.device.type != "cuda" or (t.device.index if t.device.index is not None else torch.cuda.current_device()) != engine.device_index:
            raise _lib.FacError("all inputs must be on cuda:%d (no CPU fallback, no cross-device copies); got %s"
                                % (engine.device_index, t.device))


def _int_list(values, what):
    """Per-lane counts of a ragged batch, given as a sequence of ints or a 1-D integer tensor, read on the host once: a
    list of ints.  Anything else raises ValueError."""
    if isinstance(values, torch.Tensor):
        if values.dim() != 1 or values.is_floating_point() or values.is_complex() or values.dtype == torch.bool:
            raise ValueError("%s must be a 1-D integer tensor; got %s %s" % (what, values.dtype, tuple(values.shape)))
        values = values.tolist()
    try:
        values = list(values)
        vals = [operator.index(v) for v in values]
    except TypeError:
        raise ValueError("%s must hold integers" % what) from None
    if any(isinstance(v, bool) for v in values):
        raise ValueError("%s must hold integers, not booleans" % what)
    return vals


def _lane_counts(values, B, lo, hi, what):
    """_int_list(values), checked to hold B counts in [lo, hi] (ValueError otherwise)."""
    vals = _int_list(values, what)
    if len(vals) != B:
        raise ValueError("%s holds %d values for a batch of %d" % (what, len(vals), B))
    for b, v in enumerate(vals):
        if not lo <= v <= hi:
            raise ValueError("%s[%d] = %d lies outside [%d, %d]" % (what, b, v, lo, hi))
    return vals


def _c_ints(vals):
    return None if vals is None else (ctypes.c_int * len(vals))(*vals)


def _codes_args(codes, timbre, check_devices, frames=None):
    """Validates the inputs of the decode-from-codes calls: ``codes`` = [codes_p [B,1,T], codes_c [B,1|2,T], codes_r
    [B,0..3,T] or None] integer tensors and ``timbre`` [B,1024]; ``check_devices`` raises FacError for tensors off the
    engine's device.  Returns (codes_p, codes_c, codes_r or None, residual rows, timbre, B, T) ready for the C call.
    Out-of-range codes raise IndexError, as F.embedding does in the reference; that check is one device reduction and
    one host synchronisation.  ``frames`` (a ragged batch, see _lane_counts) must hold B counts in [1, T], and only codes
    below each lane's count are checked."""
    if not isinstance(codes, (list, tuple)) or len(codes) != 3 or codes[0] is None or codes[1] is None or timbre is None:
        raise ValueError("codes must be [codes_p, codes_c, codes_r or None] and timbre a [B, 1024] tensor")
    check_devices([t for t in (*codes, timbre) if t is not None])
    for t in codes:
        if t is not None and (t.dim() != 3 or t.is_floating_point() or t.is_complex()):
            raise ValueError("codes must be integer tensors [B, rows, T]; got %s %s" % (t.dtype, tuple(t.shape)))
    cp, cc, cr = (None if t is None else t.detach().to(torch.int64).contiguous() for t in codes)
    B, _, T = cp.shape
    for name, t, rows in (("codes_p", cp, (1,)), ("codes_c", cc, (1, 2)), ("codes_r", cr, (0, 1, 2, 3))):
        if t is not None and (t.shape[1] not in rows or t.shape[0] != B or t.shape[2] != T):
            raise ValueError("%s: expected [%d, %s, %d], got %s" % (name, B, "|".join(map(str, rows)), T, tuple(t.shape)))
    if B < 1 or T < 1:
        raise ValueError("codes hold no frames: %s" % (tuple(cp.shape),))
    if tuple(timbre.shape) != (B, 1024):
        raise ValueError("timbre must be [%d, 1024], got %s" % (B, tuple(timbre.shape)))
    if cr is not None and cr.shape[1] == 0:
        cr = None
    live = None
    if frames is not None:
        counts = torch.tensor(_lane_counts(frames, B, 1, T, "frames"), dtype=torch.int64).to(cp.device)
        live = torch.arange(T, device=cp.device).view(1, 1, T) < counts.view(B, 1, 1)
    bad = [(t < 0) | (t >= 1024) for t in (cp, cc, cr) if t is not None]
    if live is not None:
        bad = [m & live for m in bad]
    if bool(torch.stack([m.any() for m in bad]).any()):
        raise IndexError("codes must lie in [0, 1024)")
    return cp, cc, cr, 0 if cr is None else cr.shape[1], _f32c(timbre), B, T


class Encoder(_RefKeyModule):
    """dac/model/dac.py:69-104 Encoder(d_model=64, strides=[2,5,5,6], d_latent=1024, causal=True, lstm=2)."""
    _module_id = MOD_ENCODER

    def __init__(self, d_model=64, strides=(2, 5, 5, 6), d_latent=1024, causal=True, lstm=2, engine=None):
        if (d_model, tuple(strides), d_latent, bool(causal), lstm) != (64, (2, 5, 5, 6), 1024, True, 2):
            raise NotImplementedError("only the configs/config.yml encoder geometry is built")
        super().__init__(synth.synth_encoder(1), engine)
        self.enc_dim = 1024

    def forward(self, x):
        L, h = self._prep(x)
        x = _f32c(x)
        B, C, T = x.shape
        assert C == 1, "encoder expects [B,1,T]"
        z = torch.empty(B, 1024, L.fac_encode_frames(T), device=x.device, dtype=torch.float32)
        _lib.check(h, L.fac_encode(h, _ptr(x), B, T, _ptr(z), _stream(x.device)), "fac_encode")
        return z


class Decoder(_RefKeyModule):
    """dac/model/dac.py:131-165 Decoder(1024, 1536, [6,5,5,2], causal, lstm): the codec's decoder (causal=True, lstm=2,
    configs/config.yml) or the redecoder model's (causal=False, lstm=0, configs/config_redecoder.yml)."""
    _module_id = MOD_DECODER

    def __init__(self, input_channel=1024, channels=1536, rates=(6, 5, 5, 2), d_out=1, causal=True, lstm=2, engine=None):
        if (input_channel, channels, tuple(rates), d_out) != (1024, 1536, (6, 5, 5, 2), 1) or \
                (bool(causal), int(lstm)) not in ((True, 2), (False, 0)):
            raise NotImplementedError("built: the config.yml decoder (causal, lstm=2) and the config_redecoder.yml one "
                                      "(non-causal, lstm=0)")
        super().__init__(synth.synth_decoder(3, lstm=int(lstm)), engine, module_id=MOD_DECODER if causal else MOD_REDEC_DECODER)
        self.causal = bool(causal)

    def forward(self, z):
        L, h = self._prep(z)
        z = _f32c(z)
        B, C, Tf = z.shape
        assert C == 1024
        y = torch.empty(B, 1, Tf * 300, device=z.device, dtype=torch.float32)
        fn = L.fac_decode if self.causal else L.fac_redecoder_decode
        _lib.check(h, fn(h, _ptr(z), B, Tf, _ptr(y), _stream(z.device)), "fac_decode")
        return y


class Redecoder(_RefKeyModule):
    """modules/redecoder.py:5-48 Redecoder(args) with args.encoder_type == 'wavenet' (wavenet_embed_dim 512, 1 prosody + 2
    content codebooks): forward(p_code, c_code, timbre_vec, use_p_code=True, use_c_code=True, n_c=2) -> [B, 1024, T]."""
    _module_id = MOD_REDECODER

    def __init__(self, args=None, engine=None):
        def g(name, default):
            if args is None:
                return default
            return args[name] if isinstance(args, dict) and name in args else getattr(args, name, default)
        if (g("encoder_type", "wavenet"), g("wavenet_embed_dim", 512), g("n_p_codebooks", 1), g("n_c_codebooks", 2),
                bool(g("decoder_causal", False))) != ("wavenet", 512, 1, 2, False):
            raise NotImplementedError("only the configs/config_redecoder.yml geometry (wavenet, 512, 1 + 2 codebooks, non-causal)")
        super().__init__(synth.synth_redecoder(7), engine)
        self.n_p_codebooks, self.n_c_codebooks, self.codebook_size, self.embed_dim = 1, 2, 1024, 512
        self.encoder_type = "wavenet"

    def forward(self, p_code, c_code, timbre_vec, use_p_code=True, use_c_code=True, n_c=2):
        """Codes outside [0, 1024) raise IndexError, as F.embedding does (one device reduction + one host sync)."""
        cp, cc, _, _, tv, B, T = _codes_args([p_code, c_code, None], timbre_vec, lambda ts: self._prep(*ts))
        L, h = self._engine.L, self._engine.handle
        if cc.shape[1] < n_c:
            raise IndexError("c_code has %d codebooks, n_c = %d" % (cc.shape[1], n_c))
        z = torch.empty(B, 1024, T, device=cp.device, dtype=torch.float32)
        rc = L.fac_redecode(h, _ptr(cp), _ptr(cc), cc.shape[1], _ptr(tv), B, T, int(bool(use_p_code)), int(bool(use_c_code)),
                            int(n_c), _ptr(z), _stream(cp.device))
        _lib.check(h, rc, "fac_redecode")
        return z


class FAquantizer(_RefKeyModule):
    """modules/quantize.py:156-454 FAquantizer(..., separate_prosody_encoder=True, timbre_norm=True);
    forward == forward_v2 (:375-454)."""
    _module_id = MOD_QUANTIZER
    _buffer_keys = ("to_mel.spectrogram.window", "to_mel.mel_scale.fb")

    def __init__(self, in_dim=1024, n_p_codebooks=1, n_c_codebooks=2, n_t_codebooks=2, n_r_codebooks=3,
                 codebook_size=1024, codebook_dim=8, quantizer_dropout=0.5, causal=True,
                 separate_prosody_encoder=True, timbre_norm=True, engine=None):
        cfg = (in_dim, n_p_codebooks, n_c_codebooks, n_r_codebooks, codebook_size, codebook_dim, bool(causal),
               bool(separate_prosody_encoder), bool(timbre_norm))
        if cfg != (1024, 1, 2, 3, 1024, 8, True, True, True):
            raise NotImplementedError("only the configs/config.yml quantizer geometry is built")
        super().__init__(synth.synth_quantizer(2), engine)
        self.hop_length = 300
        self.is_timbre_norm = True

    def forward(self, x, wave_segments, n_c=1, n_t=2, full_waves=None, wave_lens=None, return_codes=False):
        L, h = self._prep(x, wave_segments, full_waves)
        if not (1 <= int(n_c) <= 2):
            raise ValueError("n_c must be 1 or 2 (content codebooks)")
        x = _f32c(x)
        wave = _f32c(wave_segments)
        B, C, Tz = x.shape
        T = wave.shape[-1]
        Tq = min(T // 300, Tz)
        dev = x.device
        outs = torch.empty(B, 1024, Tq, device=dev)
        zp, zc, zr = (torch.empty(B, 1024, Tq, device=dev) for _ in range(3))
        losses = torch.empty(2, device=dev)
        timbre = torch.empty(B, 1024, device=dev)
        cp = torch.empty(B, 1, Tq, device=dev, dtype=torch.int64)
        cc = torch.empty(B, n_c, Tq, device=dev, dtype=torch.int64)
        cr = torch.empty(B, 3, Tq, device=dev, dtype=torch.int64)
        fw = wl = None
        tfull = 0
        if full_waves is not None:
            fw = _f32c(full_waves)
            wl = wave_lens.detach().to(dev, torch.int64).contiguous()
            tfull = fw.shape[-1]
        rc = L.fac_quantize(h, _ptr(x), _ptr(wave), B, T, Tz, int(n_c), _ptr(fw), tfull, _ptr(wl), _ptr(outs), _ptr(zp),
                            _ptr(zc), _ptr(zr), _ptr(losses), _ptr(timbre), _ptr(cp), _ptr(cc), _ptr(cr), _stream(dev))
        _lib.check(h, rc, "fac_quantize")
        quantized = [zp, zc, zr]
        if return_codes:
            return outs, quantized, losses[0], losses[1], timbre, [cp, cc, cr]
        return outs, quantized, losses[0], losses[1], timbre

    forward_v2 = forward

    def from_codes(self, codes, timbre):
        """Latents from codes: ResidualVectorQuantize.from_codes (dac/nn/quantize.py:200-220) of the prosody, content and
        residual quantizers, then outs = LayerNorm((z_p + z_c) + z_r) * gamma + beta with gamma | beta =
        timbre_linear(timbre) (modules/quantize.py:437-449).  ``codes`` is the [codes_p, codes_c, codes_r] list
        ``forward(..., return_codes=True)`` returns; codes_c may have 1 or 2 rows, codes_r 0..3 rows or be None (then z_r is
        zeros and left out of outs).  ``timbre`` [B,1024] may come from another utterance.  Returns
        (outs [B,1024,T], [z_p, z_c, z_r]).  Out-of-range codes raise IndexError (one device reduction + one host sync)."""
        cp, cc, cr, n_r, tv, B, T = _codes_args(codes, timbre, lambda ts: self._prep(*ts))
        L, h = self._engine.L, self._engine.handle
        dev = cp.device
        outs, zp, zc, zr = (torch.empty(B, 1024, T, device=dev) for _ in range(4))
        rc = L.fac_dequantize(h, _ptr(cp), _ptr(cc), cc.shape[1], _ptr(cr), n_r, _ptr(tv), B, T, _ptr(outs), _ptr(zp), _ptr(zc),
                              _ptr(zr), _stream(dev))
        _lib.check(h, rc, "fac_dequantize")
        return outs, [zp, zc, zr]


class Munch(dict):
    """Attribute dict (the reference returns munch.Munch from build_model)."""
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


class Codec:
    """reconstruct.py:56-61 as one C call: encoder -> quantizer(n_c) -> decoder, latents resident."""

    def __init__(self, model):
        self.model = model
        self.engine = model.encoder._engine

    def forward(self, x, n_c=2, lengths=None):
        """x [B,1,T] on the GPU -> (y [B,1,T'], [codes_p, codes_c, codes_r], timbre).
        lengths: a batch of utterances of different lengths -- B sample counts in (1024, T] (ints or a 1-D integer
        tensor).  Utterance b is x[b, :, :lengths[b]]: its F_b = min(lengths[b] // 300, fac_encode_frames(lengths[b]))
        code frames, timbre and 300 F_b samples are bit-identical to its own B = 1 call; codes past F_b are -1 (a decode
        without frames rejects them) and y past 300 F_b is 0.  Samples past lengths[b] are never read."""
        e = self.engine
        for m in (self.model.encoder, self.model.quantizer, self.model.decoder):
            if m.training:
                raise NotImplementedError("eval mode only")
        e.sync_weights(x.device)
        x = _f32c(x)
        B, _, T = x.shape
        lanes = _c_ints(None if lengths is None else _lane_counts(lengths, B, 1025, T, "lengths"))
        Tq = min(T // 300, e.L.fac_encode_frames(T))
        dev = x.device
        y = torch.empty(B, 1, Tq * 300, device=dev)
        cp = torch.empty(B, 1, Tq, device=dev, dtype=torch.int64)
        cc = torch.empty(B, n_c, Tq, device=dev, dtype=torch.int64)
        cr = torch.empty(B, 3, Tq, device=dev, dtype=torch.int64)
        timbre = torch.empty(B, 1024, device=dev)
        rc = e.L.fac_codec_forward_lens(e.handle, _ptr(x), B, T, lanes, n_c, _ptr(y), _ptr(cp), _ptr(cc), _ptr(cr), _ptr(timbre),
                                        _stream(dev))
        _lib.check(e.handle, rc, "fac_codec_forward")
        return y, [cp, cc, cr], timbre

    def encode(self, x, n_c=2, lengths=None):
        """Compress only: x [B,1,T] on the GPU -> ([codes_p, codes_c, codes_r], timbre), bit-identical to what forward()
        returns, without running the decoder.  lengths: per-utterance sample counts, as forward() takes them."""
        e = self.engine
        for m in (self.model.encoder, self.model.quantizer):
            if m.training:
                raise NotImplementedError("eval mode only")
        e.sync_weights(x.device)
        x = _f32c(x)
        B, _, T = x.shape
        lanes = _c_ints(None if lengths is None else _lane_counts(lengths, B, 1025, T, "lengths"))
        Tq = min(T // 300, e.L.fac_encode_frames(T))
        dev = x.device
        cp = torch.empty(B, 1, Tq, device=dev, dtype=torch.int64)
        cc = torch.empty(B, n_c, Tq, device=dev, dtype=torch.int64)
        cr = torch.empty(B, 3, Tq, device=dev, dtype=torch.int64)
        timbre = torch.empty(B, 1024, device=dev)
        rc = e.L.fac_codec_encode_lens(e.handle, _ptr(x), B, T, lanes, n_c, _ptr(cp), _ptr(cc), _ptr(cr), _ptr(timbre),
                                       _stream(dev))
        _lib.check(e.handle, rc, "fac_codec_encode")
        return [cp, cc, cr], timbre

    def timbre(self, x, lengths=None):
        """Timbre only: x [B,1,T] on the GPU -> timbre [B,1024], encode(x, n_c, lengths)[1] bit for bit for any n_c.  It runs
        the mel front-end and the StyleEncoder alone (no encoder, prosody or VQ launch), so it is the cheap way to get a
        voice to decode or convert with.  lengths: per-utterance sample counts, as encode() takes them."""
        e = self.engine
        if self.model.quantizer.training:
            raise NotImplementedError("eval mode only")
        e.sync_weights(x.device)
        x = _f32c(x)
        B, _, T = x.shape
        lanes = _c_ints(None if lengths is None else _lane_counts(lengths, B, 1025, T, "lengths"))
        timbre = torch.empty(B, 1024, device=x.device)
        rc = e.L.fac_codec_timbre_lens(e.handle, _ptr(x), B, T, lanes, _ptr(timbre), _stream(x.device))
        _lib.check(e.handle, rc, "fac_codec_timbre")
        return timbre

    def decode(self, codes, timbre, frames=None):
        """Decompress: codes ([codes_p, codes_c, codes_r] as forward()/encode() return them, or codefile.DACFile.unpack();
        codes_r may have 0..3 rows or be None) + timbre [B,1024] on the GPU -> y [B,1,300*T].  A timbre from another
        utterance gives that voice (FAquantizer.from_codes).  Out-of-range codes raise IndexError (one device reduction +
        one host sync).
        frames: a batch of utterances of different lengths -- B frame counts in [1, T] (ints or a 1-D integer tensor).
        Utterance b is codes[..., :frames[b]]: its samples are bit-identical to its own B = 1 decode, codes past its end
        are neither read nor checked, and y[b, 0, 300 * frames[b]:] is 0."""
        if self.model.decoder.training:
            raise NotImplementedError("eval mode only")
        frames = None if frames is None else _int_list(frames, "frames")
        cp, cc, cr, n_r, tv, B, T = _codes_args(codes, timbre, lambda ts: self.model.quantizer._prep(*ts), frames)
        e = self.engine
        dev = cp.device
        y = torch.empty(B, 1, T * 300, device=dev)
        lanes = _c_ints(frames)
        rc = e.L.fac_codes_decode_lens(e.handle, _ptr(cp), _ptr(cc), cc.shape[1], _ptr(cr), n_r, _ptr(tv), B, T, lanes,
                                       _ptr(y), _stream(dev))
        _lib.check(e.handle, rc, "fac_codes_decode")
        return y

    def forward_host(self, x_host, n_c=2, out=None):
        """End-to-end with HOST tensors (pinned recommended): H2D, forward, D2H inside the call.
        x_host [B,1,T] float32 CPU -> (y_host [B,1,T'], [codes_p, codes_c, codes_r]) CPU tensors."""
        e = self.engine
        dev = torch.device("cuda", torch.cuda.current_device() if e.device_index is None else e.device_index)
        e.sync_weights(dev)
        assert x_host.device.type == "cpu" and x_host.dtype == torch.float32 and x_host.is_contiguous()
        B, _, T = x_host.shape
        Tq = min(T // 300, e.L.fac_encode_frames(T))
        if out is None:
            pin = torch.cuda.is_available()
            out = (torch.empty(B, 1, Tq * 300, pin_memory=pin),
                   torch.empty(B, 1, Tq, dtype=torch.int64, pin_memory=pin),
                   torch.empty(B, n_c, Tq, dtype=torch.int64, pin_memory=pin),
                   torch.empty(B, 3, Tq, dtype=torch.int64, pin_memory=pin))
        y, cp, cc, cr = out
        with torch.cuda.device(dev):
            rc = e.L.fac_codec_forward_host(e.handle, _ptr(x_host), B, T, n_c, _ptr(y), _ptr(cp), _ptr(cc), _ptr(cr), _stream(dev))
        _lib.check(e.handle, rc, "fac_codec_forward_host")
        return y, [cp, cc, cr]

    def forward_graphed(self, x, n_c=2):
        """The same call replayed from a CUDA graph (one graph per (B, T, n_c, device), captured on first use after one
        eager call has sized the workspace): for latency-bound shapes (B = 1: 115 launches, two of them cooperative LSTM
        layers, plus the forked quantizer front) the launches leave the host in one go.  Returns the graph's OWN output
        tensors: they are overwritten by the next replay of the same shape -- clone what must survive."""
        x = _f32c(x)
        key = (tuple(x.shape), int(n_c), x.device.index)
        if not hasattr(self, "_graphs"):
            self._graphs = {}
        ent = self._graphs.get(key)
        if ent is None:
            self.forward(x, n_c)                                  # sizes the workspace, creates the side stream (not capturable)
            torch.cuda.synchronize(x.device)
            sx = x.clone()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = self.forward(sx, n_c)
            ent = self._graphs[key] = (g, sx, out, self.launch_count())
        g, sx, out, _ = ent
        sx.copy_(x)
        g.replay()
        return out

    def launch_count(self):
        return self.engine.L.fac_last_launch_count(self.engine.handle)


class CodecStream:
    """Chunked (streaming) use of the causal encoder / decoder of a build_model() Munch (README.md:105-107): feeding an
    utterance in pieces gives the results of ONE offline model.encoder(x) / model.decoder(z) call (dac/model/dac.py:103-104,
    :164-165).  The conv left context and the SLSTM (h, c) states live on the device between calls (fac_stream_*)."""

    def __init__(self, model, batch, device=None):
        self.model = model
        self.engine = model.encoder._engine
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.engine.sync_weights(dev)
        self.device = torch.device("cuda", self.engine.device_index)
        self.batch = int(batch)
        sid = self.engine.L.fac_stream_begin(self.engine.handle, self.batch)
        _lib.check(self.engine.handle, sid, "fac_stream_begin")
        self.sid = sid
        self._n_c = 0   # content codebooks of encode_codes (fixed by its first call)

    def _check(self, t):
        if t.device.type != "cuda" or (t.device.index if t.device.index is not None else torch.cuda.current_device()) != self.engine.device_index:
            raise _lib.FacError("stream inputs must be on cuda:%d (no CPU fallback); got %s" % (self.engine.device_index, t.device))
        if self.sid is None:
            raise _lib.FacError("stream is closed")

    def encode(self, x):
        """x chunk [B,1,T] (T a multiple of 300; first chunk >= 3000 samples) -> z chunk [B,1024,T/300]."""
        self._check(x)
        x = _f32c(x)
        B, C, T = x.shape
        assert C == 1 and B == self.batch
        z = torch.empty(B, 1024, max(T // 300, 0), device=x.device, dtype=torch.float32)
        e = self.engine
        _lib.check(e.handle, e.L.fac_stream_encode(e.handle, self.sid, _ptr(x), T, _ptr(z), _stream(x.device)), "fac_stream_encode")
        return z

    def decode(self, z):
        """z chunk [B,1024,Fc] (first chunk >= 10 frames) -> y chunk [B,1,300*Fc]."""
        self._check(z)
        z = _f32c(z)
        B, C, Fc = z.shape
        assert C == 1024 and B == self.batch
        y = torch.empty(B, 1, Fc * 300, device=z.device, dtype=torch.float32)
        e = self.engine
        _lib.check(e.handle, e.L.fac_stream_decode(e.handle, self.sid, _ptr(z), Fc, _ptr(y), _stream(z.device)), "fac_stream_decode")
        return y

    def decode_codes(self, codes, timbre):
        """decode() from a chunk of codes ([codes_p, codes_c, codes_r] of Fc frames, as Codec.decode takes them) and the
        utterance's timbre [B,1024] -> y chunk [B,1,300*Fc].  It advances the same decoder state as decode(): feed a stream
        one or the other."""
        def check(ts):
            for t in ts:
                self._check(t)
        cp, cc, cr, n_r, tv, B, Fc = _codes_args(codes, timbre, check)
        if B != self.batch:
            raise ValueError("stream batch is %d, codes have %d utterances" % (self.batch, B))
        y = torch.empty(B, 1, Fc * 300, device=cp.device, dtype=torch.float32)
        e = self.engine
        rc = e.L.fac_stream_decode_codes(e.handle, self.sid, _ptr(cp), _ptr(cc), cc.shape[1], _ptr(cr), n_r, _ptr(tv), Fc, _ptr(y),
                                         _stream(cp.device))
        _lib.check(e.handle, rc, "fac_stream_decode_codes")
        return y

    def encode_codes(self, x, n_c=2):
        """Compress a chunk: x [B,1,T] (T a multiple of 300; first chunk >= 3000 samples) -> [codes_p [B,1,F], codes_c
        [B,n_c,F], codes_r [B,3,F]] int64, F = T/300 - 1 on the first call and T/300 after it.  The codes run one frame
        behind the samples (the last mel frame reads 300 samples past the chunk; finish_codes() emits it), and n_c is fixed
        by the first call.  Concatenated with finish_codes(), the codes equal Codec.encode(x, n_c) on the whole utterance
        bit for bit.  A stream is fed either encode() or encode_codes(); decode_codes() runs on its own decoder state and
        may consume these codes as they come out (with any timbre)."""
        self._check(x)
        x = _f32c(x)
        B, C, T = x.shape
        assert C == 1 and B == self.batch
        F = max(T // 300 - (self._n_c == 0), 1)      # the first call holds back one frame
        dev = x.device
        cp = torch.empty(B, 1, F, device=dev, dtype=torch.int64)
        cc = torch.empty(B, n_c, F, device=dev, dtype=torch.int64)
        cr = torch.empty(B, 3, F, device=dev, dtype=torch.int64)
        e = self.engine
        rc = e.L.fac_stream_encode_codes(e.handle, self.sid, _ptr(x), T, int(n_c), _ptr(cp), _ptr(cc), _ptr(cr), _stream(dev))
        _lib.check(e.handle, rc, "fac_stream_encode_codes")
        self._n_c = int(n_c)
        return [cp, cc, cr]

    def finish_codes(self):
        """End of the utterance: ([codes_p, codes_c, codes_r] of the one held-back frame, timbre [B,1024]).  The timbre is
        Codec.encode's, bit for bit (the StyleEncoder pools over every mel frame, so it exists only now).  Closes the
        encoder half of the stream; the decoder half stays usable."""
        if self.sid is None:
            raise _lib.FacError("stream is closed")
        e = self.engine
        dev = self.device
        B = self.batch
        n_c = max(self._n_c, 1)
        cp = torch.empty(B, 1, 1, device=dev, dtype=torch.int64)
        cc = torch.empty(B, n_c, 1, device=dev, dtype=torch.int64)
        cr = torch.empty(B, 3, 1, device=dev, dtype=torch.int64)
        timbre = torch.empty(B, 1024, device=dev)
        rc = e.L.fac_stream_finish_codes(e.handle, self.sid, _ptr(cp), _ptr(cc), _ptr(cr), _ptr(timbre), _stream(dev))
        _lib.check(e.handle, rc, "fac_stream_finish_codes")
        return [cp, cc, cr], timbre

    def timbre(self):
        """The timbre so far [B,1024], without ending the stream: what finish_codes() would return if the utterance ended
        now, i.e. Codec.encode(x_so_far)[1] bit for bit with x_so_far every sample fed to encode_codes.  Codes and the
        timbre emitted later do not change.  Raises FacError before the first encode_codes chunk, on a stream fed by
        encode(), after finish_codes(), and with tensor_cores < 2; the stream stays as it was."""
        if self.sid is None:
            raise _lib.FacError("stream is closed")
        e = self.engine
        timbre = torch.empty(self.batch, 1024, device=self.device)
        rc = e.L.fac_stream_timbre(e.handle, self.sid, _ptr(timbre), _stream(self.device))
        _lib.check(e.handle, rc, "fac_stream_timbre")
        return timbre

    def close(self):
        if self.sid is not None and self.engine.handle is not None:
            self.engine.L.fac_stream_end(self.engine.handle, self.sid)
        self.sid = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class VoiceConverter:
    """reconstruct_redecoder.py:118-121 as one C call: z = model.encoder(codes[0], codes[1], timbre, use_p_code, n_c);
    wave = model.decoder(z) on a build_model(stage='redecoder') Munch, latents resident."""

    def __init__(self, model):
        self.model = model
        self.engine = model.encoder._engine

    def convert(self, codes, timbre, use_p_code=False, use_c_code=True, n_c=1, frames=None):
        """codes[0] [B,1,T], codes[1] [B,1|2,T] (codes[2] is not read), timbre [B,1024] -> y [B,1,300 T].  Codes outside
        [0, 1024) raise IndexError, as F.embedding does (one device reduction + one host sync).  frames: utterances of
        different lengths in one batch, as Codec.decode takes them; each is bit-identical to its own B = 1 convert."""
        e = self.engine
        frames = None if frames is None else _int_list(frames, "frames")
        cp, cc, _, _, tv, B, T = _codes_args([codes[0], codes[1], None], timbre, lambda ts: _engine_inputs(e, ts), frames)
        dev = cp.device
        y = torch.empty(B, 1, T * 300, device=dev)
        lanes = _c_ints(frames)
        rc = e.L.fac_voice_convert_lens(e.handle, _ptr(cp), _ptr(cc), cc.shape[1], _ptr(tv), B, T, int(bool(use_p_code)),
                                        int(bool(use_c_code)), int(n_c), lanes, _ptr(y), _stream(dev))
        _lib.check(e.handle, rc, "fac_voice_convert")
        return y


class VoiceConversionStream:
    """Voice conversion in chunks (reconstruct_redecoder.py:118-121 on a live signal): codes in, converted audio out, with
    the concatenated output bit-identical to ONE VoiceConverter.convert(codes, timbre, use_p_code, use_c_code, n_c) on the
    whole utterance.  ``redecoder_model`` is a build_model(stage='redecoder') Munch; ``timbre`` [batch, 1024] (the target
    voice, e.g. Codec.encode of a reference clip) holds until set_timbre() switches it.  The redecoder and its decoder are non-causal, so
    output frame t comes out once code frames up to t + lookahead_frames (44 frames, 550 ms) are in; finish() flushes the
    rest.  The codes and latents those windows need live on the device between calls (fac_vc_stream_*)."""

    def __init__(self, redecoder_model, batch, timbre, use_p_code=False, use_c_code=True, n_c=1):
        self.model = redecoder_model
        self.engine = e = redecoder_model.encoder._engine
        self.sid = None
        self.batch = int(batch)
        _engine_inputs(e, [timbre])
        self.device = torch.device("cuda", e.device_index)
        self._timbre = _f32c(timbre)          # kept alive until the cond layer has read it; the shape check of convert()
        if tuple(self._timbre.shape) != (self.batch, 1024):
            raise ValueError("timbre must be [%d, 1024], got %s" % (self.batch, tuple(self._timbre.shape)))
        self.lookahead_frames = e.L.fac_vc_stream_lookahead()
        sid = e.L.fac_vc_stream_begin(e.handle, self.batch, _ptr(self._timbre), int(bool(use_p_code)), int(bool(use_c_code)),
                                      int(n_c), _stream(self.device))
        _lib.check(e.handle, sid, "fac_vc_stream_begin")
        self.sid = sid

    def _check(self, tensors):
        if self.sid is None:
            raise _lib.FacError("stream is closed")
        _engine_inputs(self.engine, tensors)

    def convert(self, codes):
        """codes[0] [B,1,F] and codes[1] [B,1|2,F] (a chunk of CodecStream.encode_codes, or codes as VoiceConverter.convert
        takes them; codes[2] is not read), F >= 1 -> y [B,1,300 k]: the next k converted frames, 0 <= k <= F (k = 0 until
        lookahead_frames frames are in).  Codes outside [0, 1024) raise IndexError (one device reduction + one host sync)."""
        if len(codes) < 2 or codes[0].dim() != 3 or codes[0].shape[0] != self.batch:
            raise ValueError("codes must be [codes_p [%d, 1, F], codes_c [%d, 1|2, F], ...]" % (self.batch, self.batch))
        cp, cc, _, _, _, B, F = _codes_args([codes[0], codes[1], None], self._timbre, self._check)
        e = self.engine
        y = torch.empty(B * 300 * F, device=self.device)
        k = e.L.fac_vc_stream_convert(e.handle, self.sid, _ptr(cp), _ptr(cc), cc.shape[1], F, _ptr(y), _stream(self.device))
        _lib.check(e.handle, k, "fac_vc_stream_convert")
        return y[:B * 300 * k].view(B, 1, 300 * k)

    def finish(self):
        """End of the utterance -> y [B,1,300 k], the last k <= lookahead_frames frames."""
        if self.sid is None:
            raise _lib.FacError("stream is closed")
        e = self.engine
        B = self.batch
        y = torch.empty(B * 300 * self.lookahead_frames, device=self.device)
        k = e.L.fac_vc_stream_finish(e.handle, self.sid, _ptr(y), _stream(self.device))
        _lib.check(e.handle, k, "fac_vc_stream_finish")
        return y[:B * 300 * k].view(B, 1, 300 * k)

    def set_timbre(self, timbre):
        """Converts to ``timbre`` [batch, 1024] from the next convert() on, e.g. when the caller picks another voice mid-call.
        Every sample emitted from then on, finish() included, equals VoiceConverter.convert of the whole utterance with the
        new timbre at the same positions, and everything emitted before equals it with the old one: the next call recomputes
        the latents the decoder still reads from the codes the stream keeps, so no look-ahead is lost.  A wrong shape or
        device, or a finished or closed stream, raises and changes nothing."""
        if self.sid is None:
            raise _lib.FacError("stream is closed")
        d = timbre.device
        if d.type != "cuda" or (d.index if d.index is not None else torch.cuda.current_device()) != self.engine.device_index:
            raise _lib.FacError("timbre must be on cuda:%d (no CPU fallback); got %s" % (self.engine.device_index, d))
        tv = _f32c(timbre)
        if tuple(tv.shape) != (self.batch, 1024):
            raise ValueError("timbre must be [%d, 1024], got %s" % (self.batch, tuple(tv.shape)))
        e = self.engine
        _lib.check(e.handle, e.L.fac_vc_stream_set_timbre(e.handle, self.sid, _ptr(tv), _stream(self.device)),
                   "fac_vc_stream_set_timbre")
        self._timbre = tv

    def close(self):
        if self.sid is not None and self.engine.handle is not None:
            self.engine.L.fac_vc_stream_end(self.engine.handle, self.sid)
        self.sid = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def _ptr_array(ctype, items):
    return (ctype * max(len(items), 1))(*items)


class SessionState:
    """One live pool session taken out of its pool by ``export``: the C header (``header``, bytes), the slot's device state
    (``payload``, a uint8 tensor) and the pool's Python-side bookkeeping of the session (``info``: counts, and the 24 kHz
    samples a codes session at another rate holds before its first 3000).  A session opened at another sample rate carries
    its resampler session's state in ``rate``.  ``import_session`` on any pool of the same kind, model and options (any
    device, handle or process) continues it bit for bit.  ``kind`` is "codes", "vc", "dec" or "rs"."""

    _MAGIC = b"FACSESS1"

    def __init__(self, kind, header, payload, info=None, rate=None):
        self.kind = kind
        self.header = bytes(header)
        self.payload = payload
        self.info = dict(info or {})
        self.rate = rate

    @property
    def nbytes(self):
        """Bytes held: header, payload, held samples and the resampler state."""
        held = self.info.get("held")
        return (len(self.header) + self.payload.numel() + (0 if held is None else 4 * held.numel()) +
                (0 if self.rate is None else self.rate.nbytes))

    def to(self, device):
        """The same state with its tensors on ``device`` (import_session also moves them itself)."""
        info = {k: v.to(device) if torch.is_tensor(v) else v for k, v in self.info.items()}
        return SessionState(self.kind, self.header, self.payload.to(device), info, None if self.rate is None else self.rate.to(device))

    def cpu(self):
        return self.to("cpu")

    def to_bytes(self):
        """A self-contained byte string (waits for the export to land): for parking a session or handing it to another
        process.  SessionState.from_bytes reads it back."""
        held = self.info.get("held")
        nested = b"" if self.rate is None else self.rate.to_bytes()
        meta = json.dumps({"kind": self.kind, "info": {k: v for k, v in self.info.items() if not torch.is_tensor(v)},
                           "header": len(self.header), "payload": self.payload.numel(),
                           "held": None if held is None else held.numel(), "rate": len(nested)}).encode()
        parts = [self._MAGIC, struct.pack("<Q", len(meta)), meta, self.header, self.payload.cpu().numpy().tobytes()]
        if held is not None:
            parts.append(held.detach().to("cpu", torch.float32).contiguous().numpy().tobytes())
        parts.append(nested)
        return b"".join(parts)

    @classmethod
    def from_bytes(cls, b):
        """The state to_bytes wrote, its tensors on the CPU; ValueError for anything else or a truncated string."""
        b = bytes(b)
        if b[:8] != cls._MAGIC or len(b) < 16:
            raise ValueError("not a facodec_b200 session state")
        (n,) = struct.unpack("<Q", b[8:16])
        try:
            meta = json.loads(b[16:16 + n].decode())
            o = 16 + n
            hb, pb, nh, nr = int(meta["header"]), int(meta["payload"]), meta["held"], int(meta["rate"])
        except (ValueError, KeyError, TypeError, UnicodeDecodeError) as exc:
            raise ValueError("corrupt session state: %s" % exc) from None
        need = o + hb + pb + (0 if nh is None else 4 * int(nh)) + nr
        if len(b) != need:
            raise ValueError("session state of %d bytes, its framing says %d" % (len(b), need))
        header = b[o:o + hb]
        o += hb
        payload = torch.frombuffer(bytearray(b[o:o + pb]), dtype=torch.uint8) if pb else torch.empty(0, dtype=torch.uint8)
        o += pb
        info = dict(meta["info"])
        if nh is not None:
            info["held"] = torch.frombuffer(bytearray(b[o:o + 4 * nh]), dtype=torch.float32) if nh else torch.empty(0)
            o += 4 * nh
        rate = cls.from_bytes(b[o:o + nr]) if nr else None
        return cls(meta["kind"], header, payload, info, rate)


class _StreamPool:
    """Shared plumbing of the stream pools: session bookkeeping, pointer tables, session export / import and the pool's
    lifetime."""

    _kind = None
    _rs_quantum = 1           # the quantum of the pool's resampler (sessions at other sample rates)

    def _setup(self, engine, pid):
        self.engine, self.pid = engine, pid
        self.device = torch.device("cuda", engine.device_index)
        self._open = set()
        self._rs = None           # sessions at other sample rates: one ResamplePool, made on the first such session
        self._rate = {}           # session -> its ResamplePool session

    def _rate_open(self, sample_rate, to_24k, quantum, open_session):
        """Opens a session with open_session(); one at a sample rate other than 24 kHz also gets a resampler session
        (sample_rate -> 24 kHz when to_24k, else 24 kHz -> sample_rate).  Returns (session, resampler session or None)."""
        if self.pid is None:
            raise _lib.FacError("pool is closed")
        sr = operator.index(sample_rate)
        rs = None
        if sr != 24000:
            if self._rs is None:
                self._rs = ResamplePool(self.capacity, quantum, device=self.device, engine=self.engine)
            rs = self._rs.open(sr, 24000) if to_24k else self._rs.open(24000, sr)
        try:
            s = open_session()
        except Exception:
            if rs is not None:
                self._rs.close(rs)
            raise
        if rs is not None:
            self._rate[s] = rs
        return s, rs

    def _sessions(self, sessions):
        if self.pid is None:
            raise _lib.FacError("pool is closed")
        sessions = [int(s) for s in sessions]
        for s in sessions:
            if s not in self._open:
                raise _lib.FacError("session %d is not open in this pool" % s)
        if len(set(sessions)) != len(sessions):
            raise ValueError("a step names each session at most once")
        return sessions

    def _check_device(self, t):
        if t.device.type != "cuda" or (t.device.index if t.device.index is not None else torch.cuda.current_device()) != self.engine.device_index:
            raise _lib.FacError("pool inputs must be on cuda:%d (no CPU fallback); got %s" % (self.engine.device_index, t.device))

    def export(self, sessions):
        """{session: SessionState} of the named sessions, which stay open and unchanged: export, import_session elsewhere,
        then close(session) moves a session; importing a state twice forks it.  One launch per state region for all the
        sessions (the payloads are written on the pool's device, in stream order).  A session that is unknown, closed or
        finished raises, and nothing is exported."""
        sessions = self._sessions(sessions)
        for s in sessions:
            self._check_export(s)
        states = self._export_states(sessions)
        rate = [s for s in sessions if s in self._rate]
        if rate:
            got = self._rs._export_states([self._rate[s] for s in rate])
            for s in rate:
                states[s].rate = got[self._rate[s]]
        return states

    def import_session(self, state):
        """Opens a session holding ``state`` (from export on a pool of the same kind, model and options: any device, handle
        or process) and returns its id.  From then on it produces, bit for bit, what the exported session would have from
        the same inputs, and it shares batches with the pool's other sessions.  The payload is moved to the pool's device
        here.  Raises ValueError or FacError, and changes nothing, for a state of another kind, format version, weights,
        options, pool n_c or quantum, a corrupt or truncated state, or a full pool."""
        if self.pid is None:
            raise _lib.FacError("pool is closed")
        if not isinstance(state, SessionState):
            raise ValueError("import_session takes a SessionState, got %s" % type(state).__name__)
        if state.kind != self._kind:
            raise ValueError("a %r session state cannot join a %r pool" % (state.kind, self._kind))
        s = self._import_state(state)
        if state.rate is not None:
            try:
                if self._rs is None:
                    self._rs = ResamplePool(self.capacity, self._rs_quantum, device=self.device, engine=self.engine)
                r = self._rs.import_session(state.rate)
            except Exception:
                e = self.engine
                getattr(e.L, "fac_%s_pool_close" % self._kind)(e.handle, self.pid, s)
                raise
            self._rate[s] = r
        self._open.add(s)
        self._adopt(s, state.info)
        return s

    def _check_export(self, s):
        """Raises for a session that cannot be exported (the C call checks the rest)."""

    def _info(self, s):
        """The Python-side bookkeeping of session s, as a SessionState carries it."""
        return {}

    def _adopt(self, s, info):
        """Takes over an imported session's Python-side bookkeeping."""

    def _export_states(self, sessions):
        """{session: SessionState} from one C export call over this pool's own slots."""
        e, L, n = self.engine, self.engine.L, len(sessions)
        hb, pb = ctypes.c_size_t(), ctypes.c_size_t()
        headers, payloads = [], []
        for s in sessions:
            _lib.check(e.handle, getattr(L, "fac_%s_pool_export_size" % self._kind)(e.handle, self.pid, s, ctypes.byref(hb),
                                                                                      ctypes.byref(pb)), "pool export")
            headers.append(ctypes.create_string_buffer(hb.value))
            payloads.append(torch.empty(pb.value, dtype=torch.uint8, device=self.device))
        rc = getattr(L, "fac_%s_pool_export" % self._kind)(
            e.handle, self.pid, n, _ptr_array(ctypes.c_int, sessions), _ptr_array(ctypes.c_void_p, [ctypes.addressof(h) for h in headers]),
            _ptr_array(ctypes.c_void_p, [p.data_ptr() if p.numel() else None for p in payloads]), _stream(self.device))
        _lib.check(e.handle, rc, "fac_%s_pool_export" % self._kind)
        return {s: SessionState(self._kind, headers[i].raw, payloads[i], self._info(s)) for i, s in enumerate(sessions)}

    def _import_state(self, state):
        """One C import of state's header and payload (moved to the pool's device) -> the new session id."""
        payload = state.payload.to(self.device, torch.uint8).contiguous().view(-1)
        header = ctypes.create_string_buffer(state.header, len(state.header))
        e = self.engine
        rc = getattr(e.L, "fac_%s_pool_import" % self._kind)(e.handle, self.pid, header, len(state.header),
                                                            _ptr(payload) if payload.numel() else None, payload.numel(),
                                                            _stream(self.device))
        return _lib.check(e.handle, rc, "fac_%s_pool_import" % self._kind)

    def close(self, session=None):
        """close(s) frees session s's slot; close() frees the pool."""
        e = self.engine
        if session is not None:
            s = self._sessions([session])[0]
            _lib.check(e.handle, getattr(e.L, "fac_%s_pool_close" % self._kind)(e.handle, self.pid, s), "pool close")
            self._open.discard(s)
            if s in self._rate:
                self._rs.close(self._rate.pop(s))
            self._closed(s)
            return
        if self._rs is not None:
            self._rs.close()
            self._rs = None
        self._rate = {}
        if self.pid is not None and e.handle is not None:
            getattr(e.L, "fac_%s_pool_destroy" % self._kind)(e.handle, self.pid)
        self.pid = None
        self._open = set()

    def _closed(self, s):
        """Drops a closed session's host-side bookkeeping."""

    def _resampled(self, outs, finish=False):
        """{session: y [1,1,k]} at 24 kHz -> the same at each rate session's own rate, in one resampler launch (finish: the
        y are the sessions' last chunks, and the result includes the resampler's flushed tail); 24 kHz sessions pass."""
        rate = {self._rate[s]: y for s, y in outs.items() if s in self._rate}
        if not rate:
            return outs
        got = self._rs.finish(rate) if finish else self._rs.push(rate)
        return {s: got[self._rate[s]] if s in self._rate else y for s, y in outs.items()}

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class CodecStreamPool(_StreamPool):
    """Many live compression sessions (CodecStream.encode_codes with B = 1 each) stepped in shared launches: each session
    joins, feeds chunks of its own length and leaves on its own schedule, and its codes and timbre equal those of its own
    B = 1 CodecStream fed the same chunks, bit for bit (fac_codes_pool_*).  n_c is fixed for the pool."""

    _kind = "codes"
    _rs_quantum = 300

    def __init__(self, model, capacity=256, n_c=2, device=None):
        engine = model.encoder._engine
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        engine.sync_weights(dev)
        pid = engine.L.fac_codes_pool_create(engine.handle, int(capacity), int(n_c))
        _lib.check(engine.handle, pid, "fac_codes_pool_create")
        self._setup(engine, pid)
        self.capacity, self.n_c = int(capacity), int(n_c)
        self._fed = {}            # session -> 24 kHz samples encoded so far
        self._held = {}           # rate session -> 24 kHz samples not yet encoded (before its first 3000)
        self._done = set()        # sessions whose finish_codes ran (open until closed)

    def open(self, sample_rate=24000):
        """A new session id (a slot, reused after close()); raises FacError when the pool is full.  A session at another
        sample_rate (an integer in [8000, 192000], see resample()) takes chunks of any length: they are resampled to
        24 kHz on the device, and whole 300-sample frames reach the encoder once 3000 samples exist."""
        e = self.engine

        def open_session():
            return _lib.check(e.handle, e.L.fac_codes_pool_open(e.handle, self.pid, _stream(self.device)), "fac_codes_pool_open")
        s, rs = self._rate_open(sample_rate, True, 300, open_session)
        self._open.add(s)
        self._fed[s] = 0
        if rs is not None:
            self._held[s] = self._empty()
        return s

    def _closed(self, s):
        self._fed.pop(s, None)
        self._held.pop(s, None)
        self._done.discard(s)

    def _check_export(self, s):
        if s in self._done:
            raise _lib.FacError("session %d: its utterance was finished by finish_codes" % s)

    def _info(self, s):
        return {"fed": self._fed[s], "held": self._held[s]} if s in self._held else {"fed": self._fed[s]}

    def _adopt(self, s, info):
        self._fed[s] = int(info["fed"])
        if s in self._rate:
            self._held[s] = info["held"].to(self.device, torch.float32) if "held" in info else self._empty()

    def _empty(self):
        return torch.empty(0, device=self.device)

    def _no_codes(self):
        return [torch.empty(1, r, 0, device=self.device, dtype=torch.int64) for r in (1, self.n_c, 3)]

    def encode_codes(self, chunks):
        """{session: x [1,1,T]} (T per session, with the chunk rules of CodecStream.encode_codes) -> {session: [codes_p
        [1,1,F], codes_c [1,n_c,F], codes_r [1,3,F]]}, F = T/300 - 1 on a session's first chunk and T/300 after.  One
        rejected entry rejects the whole step and leaves every session as it was.
        A session opened at another sample rate takes any T >= 0; its chunks are resampled in one launch for the step, and
        F counts the whole frames its encoder is fed: 0 until its first 3000 samples at 24 kHz, then the frames that
        accumulated.  Its codes equal Codec.encode(r[..., :L]) with r = resample(x, sample_rate, 24000) of the whole
        utterance and L = 300 * (len(r) // 300), once finish_codes() has added the rest."""
        sessions = self._sessions(chunks.keys())
        rate = [s for s in sessions if s in self._rate]
        if not rate:
            return self._encode(chunks)
        for s in sessions:                  # every rule the encoder checks, before the resampler step
            x = chunks[s]
            self._check_device(x)
            if x.dim() != 3 or x.shape[0] != 1 or x.shape[1] != 1:
                raise ValueError("session %d: x must be [1, 1, T], got %s" % (s, tuple(x.shape)))
            if s in self._done:
                raise _lib.FacError("session %d: its utterance was finished by finish_codes" % s)
            T = x.shape[2]
            if s not in self._rate and (T <= 0 or T % 300 or (self._fed[s] == 0 and T < 3000)):
                raise _lib.FacError("session %d: a chunk of %d samples (a positive multiple of 300, the first >= 3000)" % (s, T))
        rs = [self._rate[s] for s in rate]
        got = self._rs.push({self._rate[s]: chunks[s] for s in rate})
        feed = {s: chunks[s] for s in sessions if s not in self._rate}
        held = {}
        for s in rate:
            y = got[self._rate[s]].view(-1)
            if self._fed[s] == 0:
                y = torch.cat([self._held[s], y])
                if y.numel() < 3000:
                    held[s] = y
                    continue
                held[s] = self._empty()
            if y.numel():
                feed[s] = y.view(1, 1, -1)
        try:
            codes = self._encode(feed) if feed else {}
        except Exception:
            self._rs._undo(rs)              # the encoder rejected the step: give the resampler sessions their samples back
            raise
        self._held.update(held)
        return {s: codes[s] if s in codes else self._no_codes() for s in sessions}

    def _encode(self, chunks):
        sessions = self._sessions(chunks.keys())
        xs, Ts, outs = [], [], []
        for s in sessions:
            x = chunks[s]
            self._check_device(x)
            if x.dim() != 3 or x.shape[0] != 1 or x.shape[1] != 1:
                raise ValueError("session %d: x must be [1, 1, T], got %s" % (s, tuple(x.shape)))
            x = _f32c(x)
            T = x.shape[2]
            F = max(T // 300, 1)      # the frames are known after the call: T/300 - 1 on a session's first chunk
            outs.append([torch.empty(r * F, device=self.device, dtype=torch.int64) for r in (1, self.n_c, 3)])
            xs.append(x)
            Ts.append(T)
        n = len(sessions)
        frames = (ctypes.c_int * max(n, 1))()
        P = lambda ts: _ptr_array(ctypes.c_void_p, [t.data_ptr() for t in ts])
        e = self.engine
        rc = e.L.fac_codes_pool_encode_codes(e.handle, self.pid, n, _ptr_array(ctypes.c_int, sessions), _ptr_array(ctypes.c_int, Ts),
                                             P(xs), P([o[0] for o in outs]), P([o[1] for o in outs]), P([o[2] for o in outs]),
                                             frames, _stream(self.device))
        _lib.check(e.handle, rc, "fac_codes_pool_encode_codes")
        for s, T in zip(sessions, Ts):
            self._fed[s] += T
        return {s: [t[:r * frames[i]].view(1, r, frames[i]) for t, r in zip(outs[i], (1, self.n_c, 3))]
                for i, s in enumerate(sessions)}

    def finish_codes(self, sessions):
        """End of the sessions' utterances -> {session: ([codes_p, codes_c, codes_r] of the held-back frame, timbre [1,1024])},
        as CodecStream.finish_codes.  A session at another sample rate first flushes its resampler and encodes the whole
        frames that remain (a tail of fewer than 300 samples is dropped), so its codes hold k >= 1 frames; an utterance
        that resamples to fewer than 3000 samples raises FacError, as a short first chunk does."""
        sessions = self._sessions(sessions)
        rate = [s for s in sessions if s in self._rate]
        if not rate:
            return self._finish(sessions)
        for s in sessions:                  # the finish's rules, before the resampler and encoder steps
            if s in self._done:
                raise _lib.FacError("session %d: its utterance is already finished" % s)
            n = self._fed[s]
            if s in self._rate:
                n += self._held[s].numel() + self._rs.pending(self._rate[s])
            if self._fed[s] == 0 and n // 300 * 300 < 3000:
                raise _lib.FacError("session %d: %d samples at 24 kHz, fewer than the 3000 a stream starts with" % (s, n))
        rs = [self._rate[s] for s in rate]
        tails = self._rs.finish(rs)
        feed = {}
        for s in rate:
            y = torch.cat([self._held[s], tails[self._rate[s]].view(-1)])
            whole = y.numel() // 300 * 300
            if whole:
                feed[s] = y[:whole].view(1, 1, whole)
        try:
            pre = self._encode(feed) if feed else {}
        except Exception:
            self._rs._undo(rs)
            raise
        try:
            out = self._finish(sessions)
        except Exception:
            if not pre:                     # nothing reached the encoder: the step can still be taken back whole
                self._rs._undo(rs)
            raise
        for s in rate:
            self._held[s] = self._empty()
        for s in pre:
            codes, timbre = out[s]
            out[s] = ([torch.cat([a, b], dim=2) for a, b in zip(pre[s], codes)], timbre)
        return out

    def _finish(self, sessions):
        outs = [[torch.empty(1, r, 1, device=self.device, dtype=torch.int64) for r in (1, self.n_c, 3)] for _ in sessions]
        timbres = [torch.empty(1, 1024, device=self.device) for _ in sessions]
        P = lambda ts: _ptr_array(ctypes.c_void_p, [t.data_ptr() for t in ts])
        e = self.engine
        rc = e.L.fac_codes_pool_finish_codes(e.handle, self.pid, len(sessions), _ptr_array(ctypes.c_int, sessions),
                                             P([o[0] for o in outs]), P([o[1] for o in outs]), P([o[2] for o in outs]), P(timbres),
                                             _stream(self.device))
        _lib.check(e.handle, rc, "fac_codes_pool_finish_codes")
        self._done.update(sessions)
        return {s: (outs[i], timbres[i]) for i, s in enumerate(sessions)}

    def timbre(self, sessions):
        """The timbre so far of each session, without ending any -> {session: timbre [1,1024]}, each its own B = 1
        CodecStream.timbre() fed the same chunks, bit for bit.  For a session at another sample rate, the utterance so far is
        the whole 24 kHz frames its encoder has been fed: samples still held or pending in its resampler are left out.  The
        sessions run as lanes of shared StyleEncoder batches.  A session that is finished, or whose encoder has been fed
        nothing yet (a session at another rate: before its first 3000 samples at 24 kHz), rejects the whole call, and no
        session changes."""
        sessions = self._sessions(sessions)
        for s in sessions:
            if s in self._done:
                raise _lib.FacError("session %d: its utterance was finished by finish_codes" % s)
            if self._fed[s] == 0:
                raise _lib.FacError("session %d: nothing has been encoded yet" % s)
        timbres = [torch.empty(1, 1024, device=self.device) for _ in sessions]
        e = self.engine
        rc = e.L.fac_codes_pool_timbre(e.handle, self.pid, len(sessions), _ptr_array(ctypes.c_int, sessions),
                                       _ptr_array(ctypes.c_void_p, [t.data_ptr() for t in timbres]), _stream(self.device))
        _lib.check(e.handle, rc, "fac_codes_pool_timbre")
        return dict(zip(sessions, timbres))


class VoiceConversionPool(_StreamPool):
    """Many live voice-conversion sessions (VoiceConversionStream with B = 1 each, every one with its own target timbre)
    stepped in shared launches; each session's waveform equals that of its own B = 1 VoiceConversionStream fed the same
    chunks, bit for bit (fac_vc_pool_*).  use_p_code / use_c_code / n_c are the pool's defaults; a session may open with its
    own, and sessions of different modes still share launches."""

    _kind = "vc"

    def __init__(self, redecoder_model, capacity=256, use_p_code=False, use_c_code=True, n_c=1):
        engine = redecoder_model.encoder._engine
        engine.sync_weights(torch.device("cuda", torch.cuda.current_device()))
        pid = engine.L.fac_vc_pool_create(engine.handle, int(capacity), int(bool(use_p_code)), int(bool(use_c_code)), int(n_c))
        _lib.check(engine.handle, pid, "fac_vc_pool_create")
        self._setup(engine, pid)
        self.capacity = int(capacity)
        self.use_p_code, self.use_c_code, self.n_c = bool(use_p_code), bool(use_c_code), int(n_c)
        self.lookahead_frames = engine.L.fac_vc_stream_lookahead()

    def open(self, timbre, sample_rate=24000, use_p_code=None, use_c_code=None, n_c=None):
        """A new session converting to ``timbre`` [1,1024]; raises FacError when the pool is full.  A session at another
        sample_rate gets its audio resampled from 24 kHz on the device (one launch per step for all such sessions).
        use_p_code / use_c_code / n_c (None: the pool's) set the session's conversion mode; its output equals a B = 1
        VoiceConversionStream of that mode, and it shares launches with sessions of other modes."""
        if self.pid is None:
            raise _lib.FacError("pool is closed")
        self._check_device(timbre)
        tv = _f32c(timbre)
        if tuple(tv.shape) != (1, 1024):
            raise ValueError("timbre must be [1, 1024], got %s" % (tuple(tv.shape),))
        mode = (self.use_p_code if use_p_code is None else bool(use_p_code), self.use_c_code if use_c_code is None else bool(use_c_code),
                self.n_c if n_c is None else operator.index(n_c))
        if not 0 <= mode[2] <= 2:
            raise ValueError("n_c must be 0, 1 or 2, got %d" % mode[2])
        e = self.engine

        def open_session():
            if use_p_code is None and use_c_code is None and n_c is None:
                rc = e.L.fac_vc_pool_open(e.handle, self.pid, _ptr(tv), _stream(self.device))
            else:
                rc = e.L.fac_vc_pool_open_mode(e.handle, self.pid, _ptr(tv), int(mode[0]), int(mode[1]), mode[2], _stream(self.device))
            return _lib.check(e.handle, rc, "fac_vc_pool_open")
        s, _ = self._rate_open(sample_rate, False, 1, open_session)
        self._open.add(s)
        return s

    def set_timbre(self, session, timbre):
        """Session ``session`` converts to ``timbre`` [1,1024] from its next convert() on: as VoiceConversionStream.set_timbre,
        its output from then on equals VoiceConverter.convert of its whole utterance with the new timbre, and what it emitted
        before is unchanged (at another sample rate: resample() of that 24 kHz splice).  Its next step recomputes its recent
        latents, so until then it shares launches only with other switched sessions.  The other sessions are untouched.  A
        wrong shape or device, or a session that is closed or ended by finish(), raises and changes nothing."""
        s = self._sessions([session])[0]
        self._check_device(timbre)
        tv = _f32c(timbre)
        if tuple(tv.shape) != (1, 1024):
            raise ValueError("timbre must be [1, 1024], got %s" % (tuple(tv.shape),))
        e = self.engine
        _lib.check(e.handle, e.L.fac_vc_pool_set_timbre(e.handle, self.pid, s, _ptr(tv), _stream(self.device)),
                   "fac_vc_pool_set_timbre")

    def convert(self, chunks):
        """{session: codes} (codes[0] [1,1,F], codes[1] [1,1|2,F], as VoiceConversionStream.convert takes them) -> {session:
        y [1,1,300 k]}, or [1,1,k'] at a session's own sample rate: concatenated with finish(), resample() of the 24 kHz
        output.  Codes outside [0, 1024) raise IndexError (one device reduction + one host sync for the step); one
        rejected entry rejects the whole step and leaves every session as it was."""
        return self._resampled(self._convert(chunks))

    def _convert(self, chunks):
        sessions = self._sessions(chunks.keys())
        cps, ccs, ys, Fs = [], [], [], []
        for s in sessions:
            codes = chunks[s]
            if len(codes) < 2 or codes[0].dim() != 3 or codes[0].shape[0] != 1:
                raise ValueError("session %d: codes must be [codes_p [1, 1, F], codes_c [1, 1|2, F], ...]" % s)
            cp, cc, F = self._codes(codes)
            cps.append(cp); ccs.append(cc); Fs.append(F)
            ys.append(torch.empty(300 * F, device=self.device))
        if cps and bool(torch.stack([((t < 0) | (t >= 1024)).any() for t in cps + ccs]).any()):
            raise IndexError("codes must lie in [0, 1024)")
        n = len(sessions)
        frames = (ctypes.c_int * max(n, 1))()
        P = lambda ts: _ptr_array(ctypes.c_void_p, [t.data_ptr() for t in ts])
        e = self.engine
        rc = e.L.fac_vc_pool_convert(e.handle, self.pid, n, _ptr_array(ctypes.c_int, sessions), _ptr_array(ctypes.c_int, Fs),
                                     P(cps), P(ccs), _ptr_array(ctypes.c_int, [c.shape[1] for c in ccs]), P(ys), frames,
                                     _stream(self.device))
        _lib.check(e.handle, rc, "fac_vc_pool_convert")
        return {s: ys[i][:300 * frames[i]].view(1, 1, 300 * frames[i]) for i, s in enumerate(sessions)}

    def _codes(self, codes):
        """One session's codes -> (codes_p, codes_c, F), int64 and contiguous."""
        for t in codes[:2]:
            self._check_device(t)
            if t.dim() != 3 or t.is_floating_point() or t.is_complex():
                raise ValueError("codes must be integer tensors [1, rows, F]; got %s %s" % (t.dtype, tuple(t.shape)))
        cp, cc = (t.detach().to(torch.int64).contiguous() for t in codes[:2])
        F = cp.shape[2]
        if cp.shape[:2] != (1, 1) or cc.shape[0] != 1 or cc.shape[1] not in (1, 2) or cc.shape[2] != F or F < 1:
            raise ValueError("codes must be [codes_p [1, 1, F], codes_c [1, 1|2, F]] with F >= 1; got %s, %s"
                             % (tuple(cp.shape), tuple(cc.shape)))
        return cp, cc, F

    def finish(self, sessions):
        """End of the sessions' utterances -> {session: y [1,1,300 k]}, the last k <= lookahead_frames frames (at a session's
        own sample rate: resampled, with the resampler's flushed tail)."""
        return self._resampled(self._finish(sessions), finish=True)

    def _finish(self, sessions):
        sessions = self._sessions(sessions)
        ys = [torch.empty(300 * self.lookahead_frames, device=self.device) for _ in sessions]
        frames = (ctypes.c_int * max(len(sessions), 1))()
        e = self.engine
        rc = e.L.fac_vc_pool_finish(e.handle, self.pid, len(sessions), _ptr_array(ctypes.c_int, sessions),
                                    _ptr_array(ctypes.c_void_p, [y.data_ptr() for y in ys]), frames, _stream(self.device))
        _lib.check(e.handle, rc, "fac_vc_pool_finish")
        return {s: ys[i][:300 * frames[i]].view(1, 1, 300 * frames[i]) for i, s in enumerate(sessions)}


class CodecDecodePool(_StreamPool):
    """Many live receivers decoding codes back to audio (CodecStream.decode_codes with B = 1 each, every one with its own
    timbre) stepped in shared launches; each session's audio equals that of its own B = 1 CodecStream fed the same chunks and
    timbre, bit for bit (fac_dec_pool_*).  Chunk lengths and code rows (1-2 content, 0-3 residual: the bitrate) may change
    from step to step and differ between sessions that share a batch.  The decoder is causal, so every frame is final when
    it arrives; finish() only flushes the resampler of a session at another sample rate."""

    _kind = "dec"

    def __init__(self, model, capacity=256, device=None):
        engine = model.decoder._engine
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        engine.sync_weights(dev)
        pid = engine.L.fac_dec_pool_create(engine.handle, int(capacity))
        _lib.check(engine.handle, pid, "fac_dec_pool_create")
        self._setup(engine, pid)
        self.capacity = int(capacity)
        self._finished = set()    # sessions whose finish() ran (open until closed)

    def _closed(self, s):
        self._finished.discard(s)

    def _check_export(self, s):
        if s in self._finished:
            raise _lib.FacError("session %d: its code stream was ended by finish()" % s)

    def open(self, timbre, sample_rate=24000):
        """A new session decoding with ``timbre`` [1,1024]; raises FacError when the pool is full.  A session at another
        sample_rate gets its audio resampled from 24 kHz on the device (one launch per step for all such sessions)."""
        if self.pid is None:
            raise _lib.FacError("pool is closed")
        self._check_device(timbre)
        tv = _f32c(timbre)
        if tuple(tv.shape) != (1, 1024):
            raise ValueError("timbre must be [1, 1024], got %s" % (tuple(tv.shape),))
        e = self.engine

        def open_session():
            return _lib.check(e.handle, e.L.fac_dec_pool_open(e.handle, self.pid, _ptr(tv), _stream(self.device)), "fac_dec_pool_open")
        s, _ = self._rate_open(sample_rate, False, 1, open_session)
        self._open.add(s)
        return s

    def decode_codes(self, chunks):
        """{session: [codes_p [1,1,F], codes_c [1,1|2,F], codes_r [1,0..3,F] or None]} (F per session; a session's first
        chunk >= 10 frames) -> {session: y [1,1,300 F]}, or [1,1,k] at a session's own sample rate.  Codes outside [0, 1024)
        raise IndexError (one device reduction + one host sync for the step); one rejected entry rejects the whole step and
        leaves every session as it was; so does a session that finish() has ended."""
        for s in self._sessions(chunks.keys()):
            if s in self._finished:
                raise _lib.FacError("session %d: its code stream was ended by finish()" % s)
        return self._resampled(self._decode(chunks))

    def set_timbre(self, session, timbre):
        """Session ``session`` decodes with ``timbre`` [1,1024] from its next decode_codes on, e.g. the sender's own voice
        from CodecStreamPool.timbre once it exists: its audio then equals its own B = 1 CodecStream.decode_codes given that
        timbre from the same chunk on.  Its decoder state and the other sessions are untouched.  A wrong shape or device,
        or a session that is closed or ended by finish(), raises and changes nothing."""
        s = self._sessions([session])[0]
        if s in self._finished:
            raise _lib.FacError("session %d: its code stream was ended by finish()" % s)
        self._check_device(timbre)
        tv = _f32c(timbre)
        if tuple(tv.shape) != (1, 1024):
            raise ValueError("timbre must be [1, 1024], got %s" % (tuple(tv.shape),))
        e = self.engine
        _lib.check(e.handle, e.L.fac_dec_pool_set_timbre(e.handle, self.pid, s, _ptr(tv), _stream(self.device)),
                   "fac_dec_pool_set_timbre")

    def finish(self, sessions):
        """End of the sessions' code streams -> {session: y [1,1,k]}: the resampler's flushed tail of a session at another
        sample rate, empty at 24 kHz (the causal decoder itself holds nothing back).  Concatenated with its decode_codes
        outputs, a session's audio equals resample() of its 24 kHz audio.  An ended session takes no more codes until
        close()."""
        sessions = self._sessions(sessions)
        for s in sessions:
            if s in self._finished:
                raise _lib.FacError("session %d: its code stream is already ended" % s)
        outs = {s: torch.empty(1, 1, 0, device=self.device) for s in sessions}
        outs = self._resampled(outs, finish=True)
        self._finished.update(sessions)
        return outs

    def _decode(self, chunks):
        sessions = self._sessions(chunks.keys())
        cps, ccs, crs, ys = [], [], [], []
        for s in sessions:
            codes = chunks[s]
            if not isinstance(codes, (list, tuple)) or len(codes) != 3 or codes[0] is None or codes[1] is None:
                raise ValueError("session %d: codes must be [codes_p [1, 1, F], codes_c [1, 1|2, F], codes_r [1, 0..3, F] or None]" % s)
            for t in codes:
                if t is not None:
                    self._check_device(t)
                    if t.dim() != 3 or t.is_floating_point() or t.is_complex():
                        raise ValueError("codes must be integer tensors [1, rows, F]; got %s %s" % (t.dtype, tuple(t.shape)))
            cp, cc, cr = (None if t is None else t.detach().to(torch.int64).contiguous() for t in codes)
            F = cp.shape[2]
            if (cp.shape[:2] != (1, 1) or cc.shape[0] != 1 or cc.shape[1] not in (1, 2) or cc.shape[2] != F or F < 1 or
                    (cr is not None and (cr.shape[0] != 1 or cr.shape[1] > 3 or cr.shape[2] != F))):
                raise ValueError("session %d: codes must be [codes_p [1, 1, F], codes_c [1, 1|2, F], codes_r [1, 0..3, F]] with "
                                 "F >= 1; got %s" % (s, [None if t is None else tuple(t.shape) for t in codes]))
            if cr is not None and cr.shape[1] == 0:
                cr = None
            cps.append(cp); ccs.append(cc); crs.append(cr)
            ys.append(torch.empty(1, 1, 300 * F, device=self.device))
        present = [t for t in cps + ccs + crs if t is not None]
        if present and bool(torch.stack([((t < 0) | (t >= 1024)).any() for t in present]).any()):
            raise IndexError("codes must lie in [0, 1024)")
        n = len(sessions)
        P = lambda ts: _ptr_array(ctypes.c_void_p, [0 if t is None else t.data_ptr() for t in ts])
        e = self.engine
        rc = e.L.fac_dec_pool_decode_codes(e.handle, self.pid, n, _ptr_array(ctypes.c_int, sessions),
                                           _ptr_array(ctypes.c_int, [t.shape[2] for t in cps]), P(cps), P(ccs),
                                           _ptr_array(ctypes.c_int, [t.shape[1] for t in ccs]), P(crs),
                                           _ptr_array(ctypes.c_int, [0 if t is None else t.shape[1] for t in crs]), P(ys),
                                           _stream(self.device))
        _lib.check(e.handle, rc, "fac_dec_pool_decode_codes")
        return {s: ys[i] for i, s in enumerate(sessions)}


# ------------------------------------------------------------------------------------------------------------------------
# Sample-rate conversion (fac_resample*, fac_rs_pool_*): torchaudio.functional.resample with its defaults, on the device.
# ------------------------------------------------------------------------------------------------------------------------

_RS_ENGINES = {}


def _rs_geometry(orig_freq, new_freq):
    """(orig, new, width, K) of the reduced pair; ValueError for an unsupported one."""
    g = (ctypes.c_int * 4)()
    if _lib.load().fac_resample_geometry(operator.index(orig_freq), operator.index(new_freq), g) < 0:
        raise ValueError("unsupported rate pair %s -> %s: integer rates in [8000, 192000] whose reduced filter table holds "
                         "at most 65536 floats" % (orig_freq, new_freq))
    return tuple(g)


def resample_table(orig_freq, new_freq):
    """The float32 filter table [new, K] of the reduced pair, as torchaudio's _get_sinc_resample_kernel(orig_freq, new_freq,
    gcd, dtype=torch.float32) builds it (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99), step for step with the same
    torch ops on the CPU: torch's float32 sin and cos are not the C library's, and the table is meant to be torchaudio's bit
    for bit.  Equal rates give the one-tap table [[1]]."""
    o, n, width, K = _rs_geometry(orig_freq, new_freq)
    if o == n:
        return torch.ones(1, 1)
    lowpass_filter_width = 6
    base_freq = min(o, n)
    base_freq *= 0.99
    idx = torch.arange(-width, width + o, dtype=torch.float32)[None, None] / o
    t = torch.arange(0, -n, -1, dtype=torch.float32)[:, None, None] / n + idx
    t *= base_freq
    t = t.clamp_(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t *= math.pi
    scale = base_freq / o
    kernels = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kernels *= window * scale
    return kernels.reshape(n, K).contiguous()


def _rs_engine(device):
    """The engine of resample() calls on `device` (no weights: it holds the filter tables)."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    e = _RS_ENGINES.get(idx)
    if e is None:
        e = _RS_ENGINES[idx] = Engine()
        e._ensure(torch.device("cuda", idx))
    return e


def _rs_register(engine, orig_freq, new_freq):
    """Uploads the pair's filter table to the engine's device once."""
    key = _rs_geometry(orig_freq, new_freq)[:2]
    if key not in engine._rs_pairs:
        tab = resample_table(orig_freq, new_freq)
        _lib.check(engine.handle, engine.L.fac_resample_table(engine.handle, int(orig_freq), int(new_freq), _ptr(tab)),
                   "fac_resample_table")
        engine._rs_pairs.add(key)


def resample_length(orig_freq, new_freq, n):
    """Samples that n input samples resample to: ceil(new n / orig) of the reduced pair."""
    r = _lib.load().fac_resample_out_len(operator.index(orig_freq), operator.index(new_freq), operator.index(n))
    if r < 0:
        _rs_geometry(orig_freq, new_freq)
        raise ValueError("n must be >= 0")
    return r


def resample(x, orig_freq, new_freq, lengths=None):
    """torchaudio.functional.resample(x, orig_freq, new_freq) (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99) on the
    GPU: x [B,1,T] or [B,T] float on a CUDA device -> [B,1,T'] or [B,T'], T' = ceil(new T / orig) with the pair reduced by
    its gcd.  Integer rates in [8000, 192000]; equal rates copy.  Each output sums its K taps in fp32 in a fixed order, so
    it is the same bit for bit whatever batch or stream it is computed in (ResamplePool equals this call on the
    concatenated input).  Against torchaudio on the CPU the outputs agree to within float32 rounding of the same sums.
    lengths: B sample counts in [0, T]; lane b resamples x[b, ..., :lengths[b]] and is 0 past its own ceil(new n_b / orig)
    samples.  This is not librosa.load(sr=...)'s resampler (soxr, a different filter): audio loaded by librosa at 24 kHz
    and audio resampled here differ by more than rounding."""
    if x.device.type != "cuda":
        raise _lib.FacError("resample runs on CUDA tensors only (no CPU fallback); got " + str(x.device))
    if x.dim() not in (2, 3) or (x.dim() == 3 and x.shape[1] != 1):
        raise ValueError("x must be [B, 1, T] or [B, T], got %s" % (tuple(x.shape),))
    e = _rs_engine(x.device)
    _rs_register(e, orig_freq, new_freq)
    B, T = x.shape[0], x.shape[-1]
    Tout = resample_length(orig_freq, new_freq, T)
    y = torch.empty(tuple(x.shape[:-1]) + (Tout,), device=x.device)
    if B == 0 or T == 0:
        return y
    lanes = _c_ints(None if lengths is None else _lane_counts(lengths, B, 0, T, "lengths"))
    xc = _f32c(x)
    with torch.cuda.device(x.device):
        rc = e.L.fac_resample(e.handle, _ptr(xc), B, T, lanes, int(orig_freq), int(new_freq), _ptr(y), _stream(x.device))
    _lib.check(e.handle, rc, "fac_resample")
    return y


class ResamplePool(_StreamPool):
    """Many live resampler sessions, each with its own rate pair, stepped in one launch per step (fac_rs_pool_*).  A
    session's outputs, concatenated over its push() steps and finish(), equal resample() of its concatenated input bit for
    bit, whatever the chunking.  push() returns every output whose window lies inside the input so far, rounded down to a
    multiple of ``quantum``; finish() returns the rest.  The counts follow from the chunk lengths alone: no step waits for
    the device."""

    _kind = "rs"

    def __init__(self, capacity=256, quantum=1, device=None, engine=None):
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        engine = engine if engine is not None else _rs_engine(dev)
        engine._ensure(dev)
        pid = engine.L.fac_rs_pool_create(engine.handle, int(capacity), int(quantum))
        _lib.check(engine.handle, pid, "fac_rs_pool_create")
        self._setup(engine, pid)
        self.capacity, self.quantum = int(capacity), int(quantum)
        self._state = {}          # session -> [orig, new, samples pushed, outputs returned]
        self._prev = {}           # session -> its _state before its last step

    def open(self, orig_freq, new_freq):
        """A new session resampling orig_freq -> new_freq; ValueError for an unsupported pair, FacError when full."""
        if self.pid is None:
            raise _lib.FacError("pool is closed")
        e = self.engine
        _rs_register(e, orig_freq, new_freq)
        s = _lib.check(e.handle, e.L.fac_rs_pool_open(e.handle, self.pid, int(orig_freq), int(new_freq)), "fac_rs_pool_open")
        self._open.add(s)
        self._state[s] = [int(orig_freq), int(new_freq), 0, 0]
        self._prev.pop(s, None)
        return s

    def _closed(self, s):
        self._state.pop(s, None)
        self._prev.pop(s, None)

    def _info(self, s):
        return dict(zip(("orig", "new", "seen", "emitted"), self._state[s]))

    def _import_state(self, state):
        _rs_register(self.engine, state.info["orig"], state.info["new"])
        return super()._import_state(state)

    def _adopt(self, s, info):
        self._state[s] = [int(info[k]) for k in ("orig", "new", "seen", "emitted")]
        self._prev.pop(s, None)        # an imported session has no step to take back

    def _undo(self, sessions):
        """Takes back each session's last push or finish (fac_rs_pool_undo): for a caller whose own step on the outputs was
        rejected.  The outputs that step returned are to be discarded."""
        sessions = self._sessions(sessions)
        e = self.engine
        _lib.check(e.handle, e.L.fac_rs_pool_undo(e.handle, self.pid, len(sessions), _ptr_array(ctypes.c_int, sessions)),
                   "fac_rs_pool_undo")
        for s in sessions:
            self._state[s] = self._prev.pop(s)

    def pending(self, session):
        """Outputs finish() would return now (known on the host)."""
        o, n, seen, emitted = self._state[session]
        return resample_length(o, n, seen) - emitted

    def _chunk(self, s, x):
        self._check_device(x)
        if x.dim() > 3 or any(d != 1 for d in x.shape[:-1]):
            raise ValueError("session %d: a chunk is [T], [1, T] or [1, 1, T], got %s" % (s, tuple(x.shape)))
        return _f32c(x).view(-1)

    def _step(self, chunks, finish):
        sessions = self._sessions(chunks.keys())
        xs = [None if chunks[s] is None else self._chunk(s, chunks[s]) for s in sessions]
        Ts = [0 if x is None else x.numel() for x in xs]
        L = self.engine.L
        counts = []
        for s, T in zip(sessions, Ts):
            o, n, seen, emitted = self._state[s]
            counts.append(resample_length(o, n, seen + T) - emitted if finish else L.fac_resample_ready(o, n, self.quantum, seen + T, emitted))
        buf = torch.empty(sum(counts), device=self.device)      # one allocation for the step's outputs
        ys = list(torch.split(buf, counts)) if counts else []
        got = (ctypes.c_int * max(len(sessions), 1))()
        P = lambda ts: _ptr_array(ctypes.c_void_p, [0 if t is None or t.numel() == 0 else t.data_ptr() for t in ts])
        e = self.engine
        fn = L.fac_rs_pool_finish if finish else L.fac_rs_pool_push
        rc = fn(e.handle, self.pid, len(sessions), _ptr_array(ctypes.c_int, sessions), _ptr_array(ctypes.c_int, Ts), P(xs), P(ys),
                got, _stream(self.device))
        _lib.check(e.handle, rc, "fac_rs_pool_finish" if finish else "fac_rs_pool_push")
        for i, s in enumerate(sessions):
            assert got[i] == counts[i], (s, got[i], counts[i])
            self._prev[s] = list(self._state[s])
            self._state[s][2] += Ts[i]
            self._state[s][3] += counts[i]
        return {s: ys[i].view(1, 1, -1) for i, s in enumerate(sessions)}

    def push(self, chunks):
        """{session: x} (x [T], [1,T] or [1,1,T] on the pool's device, any T >= 0) -> {session: y [1,1,k]}.  One rejected
        entry rejects the whole step and leaves every session as it was."""
        return self._step(chunks, False)

    def finish(self, sessions):
        """End of the sessions' input -> {session: y [1,1,k]}, the rest of each session's output.  ``sessions`` is a list,
        or a dict {session: last chunk} to push one last chunk in the same launch.  A finished session takes no more
        input; close() frees it."""
        if not isinstance(sessions, dict):
            sessions = {s: None for s in sessions}
        return self._step(sessions, True)


class _HeadLinear(nn.Module):
    """A plain nn.Linear(indim, outdim) run through the head machinery (kind "linear" of fac_head_finalize)."""

    def __init__(self, indim, outdim, seed=0, engine=None):
        super().__init__()
        self.indim, self.outdim = int(indim), int(outdim)
        g = synth._Gen(900 + seed)
        b = 1.0 / (indim ** 0.5)
        self.weight = nn.Parameter(g.uniform((outdim, indim), b), requires_grad=False)
        self.bias = nn.Parameter(g.uniform((outdim,), b), requires_grad=False)
        self._engine = engine if engine is not None else Engine()
        self._head_id = None
        self._tag = None

    def _sync(self, device):
        e = self._engine
        e._ensure(device)
        tag = (self.weight._version, self.bias._version)
        if self._tag == tag:
            return
        L, h = e.L, e.handle
        if self._head_id is None:
            self._head_id = _lib.check(h, L.fac_head_begin(h), "fac_head_begin")
        for k, p in (("linear.weight", self.weight), ("linear.bias", self.bias)):
            t = p.detach().to("cpu", torch.float32).contiguous()
            shape = (ctypes.c_int64 * t.dim())(*t.shape)
            _lib.check(h, L.fac_head_tensor(h, self._head_id, k.encode(), _ptr(t), shape, t.dim()), "fac_head_tensor(%s)" % k)
        _lib.check(h, L.fac_head_finalize(h, self._head_id, self.indim, self.outdim, 1, 2), "fac_head_finalize")
        self._tag = tag

    def forward(self, x):
        self._sync(x.device)
        e = self._engine
        x = _f32c(x)
        rows = x.numel() // self.indim
        out = torch.empty(tuple(x.shape[:-1]) + (self.outdim,), device=x.device)
        arr = (ctypes.c_void_p * 1)(out.data_ptr())
        _lib.check(e.handle, e.L.fac_head_forward(e.handle, self._head_id, _ptr(x), rows, 1, arr, _stream(x.device)), "fac_head_forward")
        return out


class FApredictors(nn.Module):
    """modules/quantize.py:456-619 FApredictors, forward only (training-side in the reference; the GradientReversal layers are
    identities in the forward pass): the f0 / phone / timbre predictors and their reversal counterparts over the quantizer's
    latents -- CNNLSTM heads (fac_head_*), one nn.Linear (timbre_predictor under timbre_norm) and the latent sums
    (fac_add3).  Same constructor flags, same state_dict keys (``rev_*_predictor.1.*`` for the heads inside nn.Sequential),
    same ``(preds, rev_preds)`` dicts; ``forward`` is ``forward_v2(quantized, timbre)`` when ``timbre_norm`` (config.yml),
    else the 4-latent ``forward(quantized)``."""

    def __init__(self, in_dim=1024, use_gr_content_f0=False, use_gr_prosody_phone=False, use_gr_residual_f0=False,
                 use_gr_residual_phone=False, use_gr_timbre_content=True, use_gr_timbre_prosody=True, use_gr_x_timbre=False,
                 norm_f0=True, timbre_norm=False, use_gr_content_global_f0=False, n_speakers=20000, engine=None):
        super().__init__()
        eng = engine if engine is not None else Engine()
        self._engine = eng
        self.in_dim = int(in_dim)
        self.flags = dict(use_gr_content_f0=use_gr_content_f0, use_gr_prosody_phone=use_gr_prosody_phone,
                          use_gr_residual_f0=use_gr_residual_f0, use_gr_residual_phone=use_gr_residual_phone,
                          use_gr_timbre_content=use_gr_timbre_content, use_gr_timbre_prosody=use_gr_timbre_prosody,
                          use_gr_x_timbre=use_gr_x_timbre, norm_f0=norm_f0, timbre_norm=timbre_norm)
        parts = OrderedDict()
        parts["f0_predictor"] = CNNLSTM(in_dim, 1, 2, seed=1, engine=eng)
        parts["phone_predictor"] = CNNLSTM(in_dim, 1024, 1, seed=2, engine=eng)
        parts["timbre_predictor"] = (_HeadLinear(in_dim, n_speakers, seed=3, engine=eng) if timbre_norm
                                     else CNNLSTM(in_dim, n_speakers, 1, global_pred=True, seed=3, engine=eng))
        parts["rev_f0_predictor.1"] = CNNLSTM(in_dim, 1, 2, seed=4, engine=eng)
        parts["rev_content_predictor.1"] = CNNLSTM(in_dim, 1024, 1, seed=5, engine=eng)
        parts["rev_timbre_predictor.1"] = CNNLSTM(in_dim, n_speakers, 1, global_pred=True, seed=6, engine=eng)
        if timbre_norm:
            parts["global_f0_predictor"] = _HeadLinear(in_dim, 1, seed=7, engine=eng)           # built, unused by forward (as in the reference)
        if use_gr_content_global_f0:
            parts["rev_global_f0_predictor.1"] = CNNLSTM(in_dim, 1, 1, global_pred=True, seed=8, engine=eng)
        self._parts = parts
        self._mods = nn.ModuleList(list(parts.values()))
        if timbre_norm:
            self.forward = self.forward_v2

    # ---- reference state_dict surface ----
    def state_dict(self, *a, prefix="", **kw):
        out = OrderedDict()
        for name, m in self._parts.items():
            if isinstance(m, _HeadLinear):
                out[prefix + name + ".weight"] = m.weight.detach()
                out[prefix + name + ".bias"] = m.bias.detach()
            else:
                out.update(m.state_dict(prefix=prefix + name + "."))
        return out

    def load_state_dict(self, sd, strict=True, assign=False):
        for name, m in self._parts.items():
            sub = {k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")}
            if isinstance(m, _HeadLinear):
                if strict and ("weight" not in sub or "bias" not in sub):
                    raise RuntimeError("missing keys: %s.weight / bias" % name)
                with torch.no_grad():
                    if "weight" in sub:
                        m.weight.copy_(sub["weight"])
                    if "bias" in sub:
                        m.bias.copy_(sub["bias"])
            else:
                m.load_state_dict(sub, strict=strict)

    def _sum(self, terms):
        """Left-to-right sum of 1-3 latents, as the reference accumulates them into zeros_like()."""
        if len(terms) == 1:
            return terms[0]
        e = self._engine
        a = [_f32c(t) for t in terms]
        out = torch.empty_like(a[0])
        _lib.check(e.handle, e.L.fac_add3(e.handle, _ptr(a[0]), _ptr(a[1]), _ptr(a[2]) if len(a) > 2 else None, a[0].numel(), _ptr(out),
                                          _stream(out.device)), "fac_add3")
        return out

    def _check(self, t):
        if self.training:
            raise NotImplementedError("eval mode only")
        if t.device.type != "cuda":
            raise _lib.FacError("FApredictors runs on CUDA tensors only (no CPU fallback)")
        self._engine._ensure(t.device)

    def forward_v2(self, quantized, timbre):
        """modules/quantize.py:564-619: quantized = [prosody, content, residual] latents [B, in_dim, T], timbre [B, in_dim]."""
        f = self.flags
        p, c, r = quantized[0], quantized[1], quantized[2]
        self._check(p)
        P = self._parts
        content_pred = P["phone_predictor"](c)[0]
        spk_pred = P["timbre_predictor"](timbre)
        f0_pred, uv_pred = P["f0_predictor"](p)
        pro_terms = ([c] if f["use_gr_content_f0"] else []) + ([r] if f["use_gr_residual_f0"] else [])
        con_terms = ([p] if f["use_gr_prosody_phone"] else []) + ([r] if f["use_gr_residual_phone"] else [])
        zeros = None
        if not pro_terms or not con_terms:
            zeros = torch.zeros_like(p)
        rev_f0_pred, rev_uv_pred = P["rev_f0_predictor.1"](self._sum(pro_terms) if pro_terms else zeros)
        rev_content_pred = P["rev_content_predictor.1"](self._sum(con_terms) if con_terms else zeros)[0]
        x_spk_pred = P["rev_timbre_predictor.1"](self._sum([p, c, r]))[0] if f["use_gr_x_timbre"] else None
        preds = {"f0": f0_pred, "uv": uv_pred, "content": content_pred, "timbre": spk_pred}
        rev_preds = {"rev_f0": rev_f0_pred, "rev_uv": rev_uv_pred, "rev_content": rev_content_pred, "x_timbre": x_spk_pred}
        return preds, rev_preds

    def forward(self, quantized):
        """modules/quantize.py:507-563 (timbre_norm = False): quantized = [prosody, content, timbre, residual] latents."""
        f = self.flags
        p, c, t, r = quantized[0], quantized[1], quantized[2], quantized[3]
        self._check(p)
        P = self._parts
        content_pred = P["phone_predictor"](c)[0]
        if f["norm_f0"]:
            spk_pred = P["timbre_predictor"](t)[0]
            f0_pred, uv_pred = P["f0_predictor"](p)
        else:
            spk_pred = P["timbre_predictor"](self._sum([t, p]))[0]
            f0_pred, uv_pred = P["f0_predictor"](self._sum([p, t]))
        pro_terms = ([c] if f["use_gr_content_f0"] else []) + ([t] if f["use_gr_timbre_prosody"] else []) + ([r] if f["use_gr_residual_f0"] else [])
        con_terms = ([p] if f["use_gr_prosody_phone"] else []) + ([t] if f["use_gr_timbre_content"] else []) + ([r] if f["use_gr_residual_phone"] else [])
        zeros = torch.zeros_like(p) if (not pro_terms or not con_terms) else None
        rev_f0_pred, rev_uv_pred = P["rev_f0_predictor.1"](self._sum(pro_terms) if pro_terms else zeros)
        rev_content_pred = P["rev_content_predictor.1"](self._sum(con_terms) if con_terms else zeros)[0]
        x_terms = [p, c, r] if f["norm_f0"] else [c, r]
        x_spk_pred = P["rev_timbre_predictor.1"](self._sum(x_terms))[0] if f["use_gr_x_timbre"] else None
        preds = {"f0": f0_pred, "uv": uv_pred, "content": content_pred, "timbre": spk_pred}
        rev_preds = {"rev_f0": rev_f0_pred, "rev_uv": rev_uv_pred, "rev_content": rev_content_pred, "x_timbre": x_spk_pred}
        return preds, rev_preds


def build_model(args=None, stage="codec", with_predictors=False):
    """Mirror of modules/commons.py:283-348 build_model(args, stage='codec') for the hot-path
    modules: returns Munch(encoder, quantizer, decoder) (the discriminator is training-only and out of scope).
    ``with_predictors=True`` adds ``fa_predictors`` (forward only) with the flags of modules/commons.py:311-322; it is
    opt-in because its two 20 000-way speaker heads are 160 MB of weights no inference call touches.
    ``args`` may be the reference's recursive_munch(config['model_params']) or None.
    stage='redecoder' returns the voice-conversion model Munch(encoder=Redecoder, decoder=Decoder(non-causal, no LSTM))."""
    if stage == "redecoder":
        # modules/commons.py:385-412: Munch(encoder=Redecoder(args), decoder=Decoder(causal=args.decoder_causal, lstm=args.decoder_lstm))
        eng = Engine()

        def ga(name, default):
            if args is None:
                return default
            return args[name] if isinstance(args, dict) and name in args else getattr(args, name, default)
        return Munch(encoder=Redecoder(args, engine=eng),
                     decoder=Decoder(input_channel=1024, channels=1536, rates=(6, 5, 5, 2), causal=ga("decoder_causal", False),
                                     lstm=ga("decoder_lstm", 0), engine=eng))
    if stage != "codec":
        raise NotImplementedError("built stages: 'codec' and 'redecoder'")

    def g(obj, name, default):
        if obj is None:
            return default
        return obj[name] if isinstance(obj, dict) and name in obj else getattr(obj, name, default)

    dac = g(args, "DAC", None)
    eng = Engine()
    encoder = Encoder(d_model=g(dac, "encoder_dim", 64), strides=tuple(g(dac, "encoder_rates", (2, 5, 5, 6))),
                      d_latent=1024, causal=g(args, "causal", True), lstm=g(args, "lstm", 2), engine=eng)
    quantizer = FAquantizer(in_dim=1024, n_p_codebooks=1, n_c_codebooks=g(args, "n_c_codebooks", 2), n_t_codebooks=2,
                            n_r_codebooks=3, codebook_size=1024, codebook_dim=8, quantizer_dropout=0.5,
                            causal=g(args, "causal", True),
                            separate_prosody_encoder=g(args, "separate_prosody_encoder", True),
                            timbre_norm=g(args, "timbre_norm", True), engine=eng)
    decoder = Decoder(input_channel=1024, channels=g(dac, "decoder_dim", 1536),
                      rates=tuple(g(dac, "decoder_rates", (6, 5, 5, 2))), causal=g(args, "causal", True),
                      lstm=g(args, "lstm", 2), engine=eng)
    out = Munch(encoder=encoder, quantizer=quantizer, decoder=decoder)
    if with_predictors:
        out["fa_predictors"] = FApredictors(in_dim=1024, use_gr_content_f0=g(args, "use_gr_content_f0", False),
                                            use_gr_prosody_phone=g(args, "use_gr_prosody_phone", False), use_gr_residual_f0=True,
                                            use_gr_residual_phone=True, use_gr_timbre_content=True,
                                            use_gr_timbre_prosody=g(args, "use_gr_timbre_prosody", False), use_gr_x_timbre=True,
                                            norm_f0=g(args, "norm_f0", True), timbre_norm=g(args, "timbre_norm", True),
                                            use_gr_content_global_f0=g(args, "use_gr_content_global_f0", True), engine=eng)
    return out


class ResidualVQ(nn.Module):
    """quantize/rvq.py:12-87 ResidualVQ over quantize/fvq.py:16-116 FactorizedVectorQuantize
    (eval forward), dim=1024 -> codebook_dim=8, 2**codebook_size entries (must be 1024).
    state_dict keys follow the reference: layers.{i}.in_proj.weight_g/_v/bias, out_proj..., _codebook.weight."""

    def __init__(self, *, num_quantizers, codebook_size=10, dim=1024, codebook_dim=8, commitment=0.25, seed=0, **kw):
        super().__init__()
        if dim != 1024 or codebook_dim != 8 or 2 ** int(codebook_size) != 1024 or not (1 <= num_quantizers <= 8):
            raise NotImplementedError("built for dim=1024, codebook_dim=8, 2**10 entries, <= 8 quantizers")
        self.num_quantizers = num_quantizers
        g = synth._Gen(1000 + seed)
        sd = OrderedDict()
        for i in range(num_quantizers):
            tmp = {}
            synth._conv(g, tmp, "in_proj", 8, 1024, 1)
            synth._conv(g, tmp, "out_proj", 1024, 8, 1)
            for k, v in tmp.items():
                v = v.squeeze(-1) if k.endswith("weight_v") else (v.reshape(-1, 1) if k.endswith("weight_g") else v)
                sd[f"layers.{i}.{k}"] = v
            sd[f"layers.{i}._codebook.weight"] = g.normal((1024, 8))
        self._keys = list(sd.keys())
        self._p = nn.ParameterDict({k.replace(".", "/"): nn.Parameter(v, requires_grad=False) for k, v in sd.items()})
        self._engine = Engine()
        self._rvq_id = None
        self._tag = None

    def state_dict(self, *a, prefix="", **kw):
        return OrderedDict((prefix + k, self._p[k.replace(".", "/")].detach()) for k in self._keys)

    def load_state_dict(self, sd, strict=True, assign=False):
        with torch.no_grad():
            for k in self._keys:
                self._p[k.replace(".", "/")].copy_(sd[k])
        self._tag = None

    def _folded(self, i, name):
        v = self._p[f"layers/{i}/{name}/weight_v"].detach().cpu().double()
        g = self._p[f"layers/{i}/{name}/weight_g"].detach().cpu().double()
        # weight_norm(nn.Linear) default dim=0: per output row
        w = (v * (g / v.norm(dim=1, keepdim=True))).float().contiguous()
        return w

    def _sync(self, device):
        e = self._engine
        e._ensure(device)
        tag = tuple(p._version for p in self._p.values())
        if self._tag == tag:
            return
        n = self.num_quantizers
        keep = []

        def arr(ts):
            keep.extend(ts)
            return (ctypes.c_void_p * n)(*[t.data_ptr() for t in ts])
        in_w = arr([self._folded(i, "in_proj") for i in range(n)])
        in_b = arr([self._p[f"layers/{i}/in_proj/bias"].detach().cpu().contiguous() for i in range(n)])
        out_w = arr([self._folded(i, "out_proj") for i in range(n)])
        out_b = arr([self._p[f"layers/{i}/out_proj/bias"].detach().cpu().contiguous() for i in range(n)])
        cb = arr([self._p[f"layers/{i}/_codebook/weight"].detach().cpu().contiguous() for i in range(n)])
        if self._rvq_id is not None:
            e.L.fac_rvq_destroy(e.handle, self._rvq_id)      # weights changed: release the previous device arena
        rid = e.L.fac_rvq_create(e.handle, n, in_w, in_b, out_w, out_b, cb)
        _lib.check(e.handle, rid, "fac_rvq_create")
        self._rvq_id, self._tag = rid, tag

    def forward(self, x, n_quantizers=None, channels_last=False, return_all=True):
        """x [B,1024,T] -> (quantized_out, indices [N,B,T], losses [N] (zeros in eval), all_quantized [N,B,1024,T])."""
        if self.training:
            raise NotImplementedError("eval mode only")
        if n_quantizers is not None and n_quantizers != self.num_quantizers:
            raise NotImplementedError("n_quantizers must equal num_quantizers")
        self._sync(x.device)
        e = self._engine
        x = _f32c(x)
        if channels_last:
            B, T, D = x.shape
        else:
            B, D, T = x.shape
        n = self.num_quantizers
        q = torch.empty_like(x)
        idx = torch.empty(n, B, T, device=x.device, dtype=torch.int64)
        allq = torch.empty((n,) + tuple(x.shape), device=x.device) if return_all else None
        rc = e.L.fac_rvq_forward(e.handle, self._rvq_id, _ptr(x), B, T, 1 if channels_last else 0, _ptr(q), _ptr(idx),
                                 _ptr(allq), _stream())
        _lib.check(e.handle, rc, "fac_rvq_forward")
        return q, idx, torch.zeros(n, device=x.device), allq


class Activation1d(nn.Module):
    """alias_free_torch/act.py:7-29 Activation1d(activation, up_ratio=2, down_ratio=2, 12, 12) with
    activation = SnakeBeta(alpha_logscale) (modules/quantize.py:29-88) or identity (activation=None)."""

    def __init__(self, channels=None, alpha_logscale=True, identity=False):
        super().__init__()
        self.identity = identity
        self.alpha_logscale = alpha_logscale
        if not identity:
            init = torch.zeros(channels) if alpha_logscale else torch.ones(channels)
            self.alpha = nn.Parameter(init.clone(), requires_grad=False)
            self.beta = nn.Parameter(init.clone(), requires_grad=False)
        self._engine = Engine()

    def forward(self, x):
        e = self._engine
        e._ensure(x.device)
        x = _f32c(x)
        B, C, T = x.shape
        y = torch.empty_like(x)
        a = b = None
        if not self.identity:
            a = (torch.exp(self.alpha) if self.alpha_logscale else self.alpha).detach().to(x.device, torch.float32).contiguous()
            b = (torch.exp(self.beta) if self.alpha_logscale else self.beta).detach().to(x.device, torch.float32).contiguous()
        rc = e.L.fac_alias_free_act(e.handle, _ptr(x), B, C, T, 0 if self.identity else 1, _ptr(a), _ptr(b), _ptr(y), _stream())
        _lib.check(e.handle, rc, "fac_alias_free_act")
        return y



class CNNLSTM(nn.Module):
    """modules/quantize.py:106-125 CNNLSTM(indim, outdim, head, global_pred=False), forward only (the FApredictors heads are
    training-side in the reference: SURVEY.md 8f rank 1).  state_dict keys follow the reference, including the registered
    Kaiser-sinc filter buffers of every Activation1d (accepted on load, regenerated on save).  forward(x [B, indim, T]) ->
    list of ``head`` tensors [B, T, outdim] ([B, outdim] when global_pred)."""

    def __init__(self, indim, outdim, head, global_pred=False, seed=0, engine=None):
        super().__init__()
        self.indim, self.outdim, self.nheads, self.global_pred = int(indim), int(outdim), int(head), bool(global_pred)
        sd = synth.synth_cnnlstm(500 + seed, self.indim, self.outdim, self.nheads)
        self._keys = list(sd.keys())
        self._p = nn.ParameterDict({k.replace(".", "/"): nn.Parameter(v, requires_grad=False) for k, v in sd.items()})
        self._engine = engine if engine is not None else Engine()
        self._head_id = None
        self._tag = None

    @staticmethod
    def _filter():
        from math import pi
        ks, half = 12, 6
        A = 2.285 * (half - 1) * pi * (4 * 0.3) + 7.95
        beta = 0.1102 * (A - 8.7) if A > 50.0 else (0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0) if A >= 21.0 else 0.0)
        win = torch.kaiser_window(ks, beta=beta, periodic=False)
        time = torch.arange(-half, half) + 0.5
        f = 2 * 0.25 * win * torch.sinc(2 * 0.25 * time)
        return (f / f.sum()).view(1, 1, ks)

    def state_dict(self, *a, prefix="", **kw):
        out = OrderedDict()
        for k in self._keys:
            out[prefix + k] = self._p[k.replace(".", "/")].detach()
            if k.endswith("act.beta"):
                base = k[:-len("act.beta")]
                out[prefix + base + "upsample.filter"] = self._filter()
                out[prefix + base + "downsample.lowpass.filter"] = self._filter()
        return out

    def load_state_dict(self, sd, strict=True, assign=False):
        missing = [k for k in self._keys if k not in sd]
        if strict and missing:
            raise RuntimeError("missing keys: %s" % missing[:5])
        with torch.no_grad():
            for k in self._keys:
                if k in sd:
                    self._p[k.replace(".", "/")].copy_(sd[k])
        self._tag = None

    def _sync(self, device):
        e = self._engine
        e._ensure(device)
        tag = tuple(p._version for p in self._p.values())
        if self._tag == tag:
            return
        L, h = e.L, e.handle
        if self._head_id is None:
            self._head_id = _lib.check(h, L.fac_head_begin(h), "fac_head_begin")
        for k in self._keys:
            t = self._p[k.replace(".", "/")].detach().to("cpu", torch.float32).contiguous()
            shape = (ctypes.c_int64 * max(t.dim(), 1))(*t.shape)
            _lib.check(h, L.fac_head_tensor(h, self._head_id, k.encode(), _ptr(t), shape, t.dim()), "fac_head_tensor(%s)" % k)
        _lib.check(h, L.fac_head_finalize(h, self._head_id, self.indim, self.outdim, self.nheads, int(self.global_pred)),
                   "fac_head_finalize")
        self._tag = tag

    def forward(self, x):
        if self.training:
            raise NotImplementedError("eval mode only")
        self._sync(x.device)
        e = self._engine
        x = _f32c(x)
        B, C, T = x.shape
        assert C == self.indim
        shape = (B, self.outdim) if self.global_pred else (B, T, self.outdim)
        outs = [torch.empty(shape, device=x.device) for _ in range(self.nheads)]
        arr = (ctypes.c_void_p * self.nheads)(*[o.data_ptr() for o in outs])
        rc = e.L.fac_head_forward(e.handle, self._head_id, _ptr(x), B, T, arr, _stream(x.device))
        _lib.check(e.handle, rc, "fac_head_forward")
        return outs


class _JdcResBlock(nn.Module):
    """Parameter holder of modules/JDC/model.py ResBlock (state-dict keys only; JDCNet.forward runs on the GPU)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.pre_conv = nn.Sequential(nn.BatchNorm2d(cin), nn.LeakyReLU(0.01), nn.MaxPool2d((1, 2)))
        self.conv = nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1, bias=False), nn.BatchNorm2d(cout), nn.LeakyReLU(0.01),
                                  nn.Conv2d(cout, cout, 3, padding=1, bias=False))
        self.conv1by1 = nn.Conv2d(cin, cout, 1, bias=False)


class JDCNet(nn.Module):
    """modules/JDC/model.py JDCNet(num_class=1, seq_len=192) -- the F0 extractor train.py loads -- in eval mode.  Same
    state-dict keys (the ``['net']`` dict of ``bst.t7``); ``forward(x, lengths=None)`` takes normalized log-mel ``x``
    [B, 1, 80, T] on a CUDA device and returns ``(F0 [B, T], GAN_feature [B, 256, 10, T], poolblock_out [B, 256, T, 2])``
    as model.py:102-137 does in eval mode.  The 3x3 convs run on the wgmma conv kernel in its fp32-faithful promoted class,
    with every BatchNorm folded in; the BiLSTM runs on the resident-weight recurrence kernel.

    ``lengths`` (B ints in [1, T]) makes a ragged batch: lane b is its own first lengths[b] frames, bit for bit what a
    B = 1 call on them returns, and its outputs past lengths[b] are zero.  The detector branch (maxpool1-3,
    detector_conv, bilstm_detector, detector) is loaded but, as in the reference forward, never run.  Training mode
    (batch statistics, dropout) raises NotImplementedError."""

    def __init__(self, num_class=1, seq_len=192, engine=None):
        super().__init__()
        if num_class != 1:
            raise ValueError("JDCNet: only num_class=1 (the F0 regressor train.py loads) is implemented")
        self.num_class, self.seq_len = num_class, seq_len
        self.conv_block = nn.Sequential(nn.Conv2d(1, 64, 3, padding=1, bias=False), nn.BatchNorm2d(64), nn.LeakyReLU(0.01),
                                        nn.Conv2d(64, 64, 3, padding=1, bias=False))
        self.res_block1 = _JdcResBlock(64, 128)
        self.res_block2 = _JdcResBlock(128, 192)
        self.res_block3 = _JdcResBlock(192, 256)
        self.pool_block = nn.Sequential(nn.BatchNorm2d(256), nn.LeakyReLU(0.01), nn.MaxPool2d((1, 4)), nn.Dropout(0.2))
        self.maxpool1 = nn.MaxPool2d((1, 40))
        self.maxpool2 = nn.MaxPool2d((1, 20))
        self.maxpool3 = nn.MaxPool2d((1, 10))
        self.detector_conv = nn.Sequential(nn.Conv2d(640, 256, 1, bias=False), nn.BatchNorm2d(256), nn.LeakyReLU(0.01),
                                           nn.Dropout(0.2))
        self.bilstm_classifier = nn.LSTM(512, 256, batch_first=True, bidirectional=True)
        self.bilstm_detector = nn.LSTM(512, 256, batch_first=True, bidirectional=True)
        self.classifier = nn.Linear(512, num_class)
        self.detector = nn.Linear(512, 2)
        for p in self.parameters():
            p.requires_grad_(False)
        self._engine = engine if engine is not None else Engine()
        self._jdc_id = None
        self._tag = None

    def _sync(self, device):
        e = self._engine
        e._ensure(device)
        sd = self.state_dict()
        tag = tuple((t._version, t.data_ptr()) for t in sd.values())
        if self._tag == tag:
            return
        L, h = e.L, e.handle
        if self._jdc_id is None:
            self._jdc_id = _lib.check(h, L.fac_jdc_begin(h), "fac_jdc_begin")
        for k, t in sd.items():
            if k.endswith("num_batches_tracked"):
                continue
            t = t.detach().to("cpu", torch.float32).contiguous()
            shape = (ctypes.c_int64 * max(t.dim(), 1))(*t.shape)
            _lib.check(h, L.fac_jdc_tensor(h, self._jdc_id, k.encode(), _ptr(t), shape, t.dim()), "fac_jdc_tensor(%s)" % k)
        _lib.check(h, L.fac_jdc_finalize(h, self._jdc_id), "fac_jdc_finalize")
        self._tag = tag

    def forward(self, x, lengths=None):
        if self.training:
            raise NotImplementedError("facodec_b200.JDCNet implements the eval-mode forward only; call .eval()")
        if not isinstance(x, torch.Tensor) or x.dim() != 4 or x.shape[1] != 1 or x.shape[2] != 80 or x.shape[3] < 1:
            raise _lib.FacError("JDCNet expects x [B, 1, 80, T]; got %s" % ((tuple(x.shape) if isinstance(x, torch.Tensor) else type(x)),))
        B, T = int(x.shape[0]), int(x.shape[3])
        if B < 1:
            raise _lib.FacError("JDCNet: empty batch")
        self._sync(x.device)
        e = self._engine
        lens = None if lengths is None else _lane_counts(lengths, B, 1, T, "lengths")
        x = _f32c(x)
        f0 = torch.empty(B, T, device=x.device)
        gan = torch.empty(B, 256, 10, T, device=x.device)
        pool = torch.empty(B, 256, T, 2, device=x.device)
        _lib.check(e.handle, e.L.fac_jdc_forward(e.handle, self._jdc_id, _ptr(x), B, T, _c_ints(lens) if lens else None, _ptr(f0),
                                                 _ptr(gan), _ptr(pool), _stream(x.device)), "fac_jdc_forward")
        return f0, gan, pool


def load_F0_models(path):
    """modules/commons.py:183-191 load_F0_models: JDCNet(num_class=1, seq_len=192) with ``torch.load(path)['net']``.
    Returned in eval mode, unlike the reference's ``.train()``: train mode uses batch statistics and dropout, so its F0
    changes from call to call; eval mode is what this package computes."""
    model = JDCNet(num_class=1, seq_len=192)
    params = torch.load(path, map_location="cpu")["net"]
    model.load_state_dict(params)
    return model.eval()


def _check_cuda(t, what):
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise _lib.FacError("%s must be a CUDA tensor (no CPU fallback); got %s" % (what, t.device if isinstance(t, torch.Tensor) else type(t)))


def f0_targets(F0, lengths=None, norm_f0=True):
    """train.py:219-251 on F0 [B, T] (CUDA): per lane, voiced = F0 > 5.0, log2, then (x - mean) / std (torch.std's unbiased
    std) on voiced frames and -10 on the others, NaN / inf replaced by -10; glob_f0 = the mean, 0 without a voiced frame
    (one voiced frame: std is NaN, so that frame is -10 and the mean is kept).  Returns (targets [B, T], glob_f0 [B]: the
    torch.stack of train.py's list); with norm_f0=False, (F0, []) as train.py leaves them.  ``lengths``: lane b's statistics cover its first
    lengths[b] frames only and the rest of its targets are -10.  Fixed-order reductions: the result does not depend on B."""
    _check_cuda(F0, "F0")
    if F0.dim() != 2:
        raise _lib.FacError("f0_targets expects F0 [B, T]; got %s" % (tuple(F0.shape),))
    if not norm_f0:
        return F0, []
    B, T = int(F0.shape[0]), int(F0.shape[1])
    lens = None if lengths is None else _lane_counts(lengths, B, 0, T, "lengths")
    x = _f32c(F0)
    out = torch.empty(B, T, device=x.device)
    glob = torch.empty(B, device=x.device)
    if B == 0 or T == 0:
        return out.fill_(-10.0), glob.zero_()
    e = _rs_engine(x.device)
    _lib.check(e.handle, e.L.fac_f0_targets(e.handle, _ptr(x), B, T, _c_ints(lens) if lens else None, _ptr(out), _ptr(glob),
                                            _stream(x.device)), "fac_f0_targets")
    return out, glob


def log_norm(x, mean=-4, std=4, dim=2):
    """modules/commons.py:176-181 log_norm: log(||exp(x * std + mean)||_2 over `dim`) for normalized log-mel x [..., 80, T]
    whose `dim` is the 80-bin axis (train.py:215: x [B, 1, 80, T], dim = 2 -> [B, 1, T]).  Only the reference's mean = -4,
    std = 4 are implemented."""
    _check_cuda(x, "x")
    if mean != -4 or std != 4:
        raise ValueError("log_norm: only mean=-4, std=4 are implemented")
    nd = x.dim()
    if nd < 2 or dim % nd != nd - 2 or x.shape[-2] != 80:
        raise _lib.FacError("log_norm expects x [..., 80, T] normed over its 80-bin axis; got %s, dim=%d" % (tuple(x.shape), dim))
    T = int(x.shape[-1])
    B = x.numel() // (80 * T) if T else 0
    xc = _f32c(x)
    out = torch.empty(tuple(x.shape[:-2]) + (T,), device=x.device)
    if B == 0 or T == 0:
        return out
    e = _rs_engine(x.device)
    _lib.check(e.handle, e.L.fac_log_norm(e.handle, _ptr(xc), B, T, _ptr(out), _stream(x.device)), "fac_log_norm")
    return out
