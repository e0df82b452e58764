"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference FAcodec
encoder -> quantizer -> decoder forward, written as plain functions over the
reference's ``state_dict`` (no nn.Module, no audiotools / munch / argbind).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` leg may import this file; the product (``facodec_b200``)
never does.

Pinning: the reference ships no tests or golden vectors (SURVEY.md section 4).
This restatement is pinned by (a) ``tests/test_oracle_vs_reference.py`` which,
inside the build container, runs the *imported unmodified reference*
(``oracle/ref_import.py``) and requires bit-identical tensors, and (b) the
fixtures under ``tests/golden/`` produced by ``oracle/make_golden.py`` from the
imported reference, which the restatement must reproduce bit-for-bit on any box.

It is fp32 torch-functional code because the reference *is* fp32 ATen code; the
same ATen kernels give the same bits.  Every function cites the reference
lines it follows (paths relative to the reference root).
"""
import math

import torch
import torch.nn.functional as F

HOP = 300


# ----------------------------------------------------------------------------
# dac/model/encodec.py
# ----------------------------------------------------------------------------
def _wn_weight(sd, prefix):
    """Legacy torch.nn.utils.weight_norm (encodec.py:42-51): w = g * v / ||v||, norm over all
    dims but 0 (for ConvTranspose1d dim 0 is in-channels)."""
    if prefix + ".weight" in sd:
        return sd[prefix + ".weight"]
    return torch._weight_norm(sd[prefix + ".weight_v"], sd[prefix + ".weight_g"], 0)


def _extra_padding(length, kernel_size, stride, padding_total):
    """encodec.py:71-78 get_extra_padding_for_conv1d."""
    n_frames = (length - kernel_size + padding_total) / stride + 1
    ideal_length = (math.ceil(n_frames) - 1) * stride + (kernel_size - padding_total)
    return ideal_length - length


def _pad1d_reflect(x, left, right):
    """encodec.py:96-113 pad1d(mode='reflect') incl. the short-input zero-extension."""
    length = x.shape[-1]
    max_pad = max(left, right)
    extra = 0
    if length <= max_pad:
        extra = max_pad - length + 1
        x = F.pad(x, (0, extra))
    padded = F.pad(x, (left, right), "reflect")
    end = padded.shape[-1] - extra
    return padded[..., :end]


def sconv1d(x, sd, prefix, stride=1, dilation=1, causal=True):
    """SConv1d.forward, encodec.py:212-228 (pad_mode='reflect'). ``prefix`` is the nn.Conv1d
    (``...conv.conv``)."""
    w = _wn_weight(sd, prefix)
    k = w.shape[-1]
    k_eff = (k - 1) * dilation + 1
    padding_total = k_eff - stride
    extra = _extra_padding(x.shape[-1], k_eff, stride, padding_total)
    if causal:
        x = _pad1d_reflect(x, padding_total, extra)
    else:
        pr = padding_total // 2
        pl = padding_total - pr
        x = _pad1d_reflect(x, pl, pr + extra)
    return F.conv1d(x, w, sd[prefix + ".bias"], stride=stride, dilation=dilation)


def sconvtr1d(x, sd, prefix, stride, causal=True):
    """SConvTranspose1d.forward, encodec.py:248-270, trim_right_ratio=1."""
    w = _wn_weight(sd, prefix)
    k = w.shape[-1]
    padding_total = k - stride
    y = F.conv_transpose1d(x, w, sd[prefix + ".bias"], stride=stride)
    if causal:
        pr = math.ceil(padding_total * 1.0)
        pl = padding_total - pr
    else:
        pr = padding_total // 2
        pl = padding_total - pr
    return y[..., pl: y.shape[-1] - pr]


def slstm(x, sd, prefix, num_layers=2):
    """SLSTM.forward, encodec.py:282-288: [B,C,T] -> [T,B,C] -> nn.LSTM(C,C,num_layers), zero
    state, + skip."""
    x = x.permute(2, 0, 1)
    B, H = x.shape[1], x.shape[2]
    flat = []
    for l in range(num_layers):
        flat += [sd[f"{prefix}.weight_ih_l{l}"], sd[f"{prefix}.weight_hh_l{l}"],
                 sd[f"{prefix}.bias_ih_l{l}"], sd[f"{prefix}.bias_hh_l{l}"]]
    h0 = torch.zeros(num_layers, B, H, dtype=x.dtype, device=x.device)
    y, _, _ = torch._VF.lstm(x, (h0, h0.clone()), flat, True, num_layers, 0.0, False, False, False)
    y = y + x
    return y.permute(1, 2, 0)


# ----------------------------------------------------------------------------
# dac/nn/layers.py, dac/model/dac.py
# ----------------------------------------------------------------------------
def snake(x, alpha):
    """dac/nn/layers.py:17-24."""
    return x + (alpha + 1e-9).reciprocal() * torch.sin(alpha * x).pow(2)


def residual_unit(x, sd, prefix, dilation, causal=True):
    """ResidualUnit, dac.py:25-42 (crop branch dead: same length)."""
    y = snake(x, sd[prefix + ".block.0.alpha"])
    y = sconv1d(y, sd, prefix + ".block.1.conv.conv", dilation=dilation, causal=causal)
    y = snake(y, sd[prefix + ".block.2.alpha"])
    y = sconv1d(y, sd, prefix + ".block.3.conv.conv", causal=causal)
    return x + y


def encoder_forward(sd, x, rates=(2, 5, 5, 6), taps=None):
    """Encoder.forward, dac.py:69-104. x [B,1,T] -> z [B,1024,ceil(T/300)]."""
    h = sconv1d(x, sd, "block.0.conv.conv")
    if taps is not None:
        taps["enc_conv0"] = h
    for i, s in enumerate(rates):
        p = f"block.{i + 1}"
        for j, d in enumerate((1, 3, 9)):
            h = residual_unit(h, sd, f"{p}.block.{j}", d)
        h = snake(h, sd[f"{p}.block.3.alpha"])
        h = sconv1d(h, sd, f"{p}.block.4.conv.conv", stride=s)
        if taps is not None:
            taps[f"enc_block{i + 1}"] = h
    n = len(rates)
    h = slstm(h, sd, f"block.{n + 1}.lstm")
    if taps is not None:
        taps["enc_lstm"] = h
    h = snake(h, sd[f"block.{n + 2}.alpha"])
    return sconv1d(h, sd, f"block.{n + 3}.conv.conv")


def decoder_forward(sd, z, rates=(6, 5, 5, 2), taps=None, causal=True, lstm=2):
    """Decoder.forward, dac.py:131-165. z [B,1024,T'] -> y [B,1,300 T'].  ``causal`` / ``lstm`` are the constructor
    arguments: the codec uses (True, 2) (configs/config.yml), the redecoder (False, 0) (configs/config_redecoder.yml:
    decoder_causal / decoder_lstm) -- without the SLSTM the nn.Sequential indices shift down by one."""
    h = sconv1d(z, sd, "model.0.conv.conv", causal=causal)
    if taps is not None:
        taps["dec_conv0"] = h
    base = 1
    if lstm:
        h = slstm(h, sd, "model.1.lstm", num_layers=lstm)
        base = 2
        if taps is not None:
            taps["dec_lstm"] = h
    for i, s in enumerate(rates):
        p = f"model.{i + base}"
        h = snake(h, sd[f"{p}.block.0.alpha"])
        h = sconvtr1d(h, sd, f"{p}.block.1.convtr.convtr", s, causal=causal)
        for j, d in enumerate((1, 3, 9)):
            h = residual_unit(h, sd, f"{p}.block.{j + 2}", d, causal=causal)
        if taps is not None:
            taps[f"dec_block{i + 1}"] = h
    n = len(rates)
    h = snake(h, sd[f"model.{n + base}.alpha"])
    h = sconv1d(h, sd, f"model.{n + base + 1}.conv.conv", causal=causal)
    return torch.tanh(h)


# ----------------------------------------------------------------------------
# mel front-end: torchaudio.transforms.MelSpectrogram as configured at
# modules/quantize.py:228-230, then preprocess :239-242
# ----------------------------------------------------------------------------
def mel_preprocess(sd, wave, n_bins=20, n_fft=2048, hop=HOP, win_length=1200):
    """wave [B,1,T] -> [B,n_bins,T//300].  torchaudio Spectrogram(center=True, reflect,
    power=2, window zero-padded to n_fft by torch.stft) -> MelScale (spec^T @ fb)^T ->
    (log(1e-5+mel)+4)/4 -> slice."""
    w = wave.squeeze(1)
    spec = torch.stft(w, n_fft, hop_length=hop, win_length=win_length,
                      window=sd["to_mel.spectrogram.window"], center=True, pad_mode="reflect",
                      normalized=False, onesided=True, return_complex=True)
    spec = spec.abs().pow(2.0)
    mel = torch.matmul(spec.transpose(-1, -2), sd["to_mel.mel_scale.fb"]).transpose(-1, -2)
    mel = (torch.log(1e-5 + mel) - (-4)) / 4
    return mel[:, :n_bins, :int(wave.size(-1) / hop)]


# ----------------------------------------------------------------------------
# modules/style_encoder.py, modules/attentions.py
# ----------------------------------------------------------------------------
def _mish(x):
    """style_encoder.py:6-10."""
    return x * torch.tanh(F.softplus(x))


def _conv1d_glu(x, sd, prefix):
    """Conv1dGLU, style_encoder.py:13-31 (padding=2 zero pad, eval => dropout off)."""
    y = F.conv1d(x, sd[prefix + ".conv1.weight"], sd[prefix + ".conv1.bias"], padding=2)
    c = y.shape[1] // 2
    x1, x2 = torch.split(y, c, dim=1)
    return x + x1 * torch.sigmoid(x2)


def _mha(x, sd, prefix, n_heads, attn_mask):
    """MultiHeadAttention.forward/attention, attentions.py:159-199, window_size=None."""
    def c1(t, n):
        return F.conv1d(t, sd[f"{prefix}.conv_{n}.weight"], sd[f"{prefix}.conv_{n}.bias"])
    q, k, v = c1(x, "q"), c1(x, "k"), c1(x, "v")
    b, d, t = k.shape
    kc = d // n_heads
    q = q.view(b, n_heads, kc, t).transpose(2, 3)
    k = k.view(b, n_heads, kc, t).transpose(2, 3)
    v = v.view(b, n_heads, kc, t).transpose(2, 3)
    scores = torch.matmul(q / math.sqrt(kc), k.transpose(-2, -1))
    scores = scores.masked_fill(attn_mask == 0, -1e4)
    p = F.softmax(scores, dim=-1)
    o = torch.matmul(p, v)
    o = o.transpose(2, 3).contiguous().view(b, d, t)
    return c1(o, "o")


def style_encoder(sd, mel, mask, prefix="timbre_encoder"):
    """StyleEncoder.forward, style_encoder.py:63-90. mel [B,80,T'], mask [B,1,T'] bool."""
    x = F.conv1d(mel, sd[prefix + ".spectral.0.weight"], sd[prefix + ".spectral.0.bias"])
    x = _mish(x)
    x = F.conv1d(x, sd[prefix + ".spectral.3.weight"], sd[prefix + ".spectral.3.bias"])
    x = _mish(x) * mask
    x = _conv1d_glu(x, sd, prefix + ".temporal.0")
    x = _conv1d_glu(x, sd, prefix + ".temporal.1") * mask
    attn_mask = mask.unsqueeze(2) * mask.unsqueeze(-1)
    x = x + _mha(x, sd, prefix + ".slf_attn", 2, attn_mask)
    x = F.conv1d(x, sd[prefix + ".fc.weight"], sd[prefix + ".fc.bias"])
    len_ = mask.sum(dim=2)
    return torch.div(x.sum(dim=2), len_)


# ----------------------------------------------------------------------------
# modules/wavenet.py
# ----------------------------------------------------------------------------
def wavenet(sd, x, prefix="melspec_encoder", hidden=256, n_layers=8, g=None, causal=True):
    """WN.forward, wavenet.py:138-166 with x_mask == 1, eval (dropout off), dilation_rate 1;
    gate = commons.py:113-120 fused_add_tanh_sigmoid_multiply.  g [B, gin, 1] (or None, the codec's own call) goes
    through cond_layer once and is sliced per layer (:143-151)."""
    output = torch.zeros_like(x)
    if g is not None:
        g = sconv1d(g, sd, f"{prefix}.cond_layer.conv.conv", causal=causal)
    for i in range(n_layers):
        x_in = sconv1d(x, sd, f"{prefix}.in_layers.{i}.conv.conv", causal=causal)
        if g is not None:
            g_l = g[:, i * 2 * hidden:(i + 1) * 2 * hidden, :]
        else:
            g_l = torch.zeros_like(x_in)
        in_act = x_in + g_l
        acts = torch.tanh(in_act[:, :hidden]) * torch.sigmoid(in_act[:, hidden:])
        rs = sconv1d(acts, sd, f"{prefix}.res_skip_layers.{i}.conv.conv", causal=causal)
        if i < n_layers - 1:
            x = (x + rs[:, :hidden]) * 1.0
            output = output + rs[:, hidden:]
        else:
            output = output + rs
    return output * 1.0


# ----------------------------------------------------------------------------
# dac/nn/quantize.py
# ----------------------------------------------------------------------------
def vq_decode_latents(latents, codebook):
    """VectorQuantize.decode_latents, dac/nn/quantize.py:78-94 (== quantize/fvq.py:101-116)."""
    b, d, t = latents.shape
    enc = latents.permute(0, 2, 1).reshape(b * t, d)
    enc = F.normalize(enc)
    cb = F.normalize(codebook)
    dist = (enc.pow(2).sum(1, keepdim=True) - 2 * enc @ cb.t() + cb.pow(2).sum(1, keepdim=True).t())
    idx = (-dist).max(1)[1].reshape(b, t)
    z_q = F.embedding(idx, codebook).transpose(1, 2)
    return z_q, idx


def vector_quantize(sd, prefix, z):
    """VectorQuantize.forward, dac/nn/quantize.py:34-70. Returns (z_q_out, commit[B], cb[B], idx, z_e)."""
    w_in = _wn_weight(sd, prefix + ".in_proj")
    z_e = F.conv1d(z, w_in, sd[prefix + ".in_proj.bias"])
    z_q, idx = vq_decode_latents(z_e, sd[prefix + ".codebook.weight"])
    commit = F.mse_loss(z_e, z_q, reduction="none").mean([1, 2])
    cbl = F.mse_loss(z_q, z_e, reduction="none").mean([1, 2])
    z_q = z_e + (z_q - z_e)
    w_out = _wn_weight(sd, prefix + ".out_proj")
    out = F.conv1d(z_q, w_out, sd[prefix + ".out_proj.bias"])
    return out, commit, cbl, idx, z_e


def residual_vq(sd, prefix, z, n_quantizers):
    """ResidualVectorQuantize.forward (eval), dac/nn/quantize.py:127-198."""
    z_q = 0
    residual = z
    commitment_loss = 0
    codebook_loss = 0
    codes, latents = [], []
    for i in range(n_quantizers):
        z_q_i, c_i, cb_i, idx_i, z_e_i = vector_quantize(sd, f"{prefix}.quantizers.{i}", residual)
        mask = torch.full((z.shape[0],), fill_value=i, device=z.device) < n_quantizers
        z_q = z_q + z_q_i * mask[:, None, None]
        residual = residual - z_q_i
        commitment_loss = commitment_loss + (c_i * mask).mean()
        codebook_loss = codebook_loss + (cb_i * mask).mean()
        codes.append(idx_i)
        latents.append(z_e_i)
    return z_q, torch.stack(codes, dim=1), torch.cat(latents, dim=1), commitment_loss, codebook_loss


# ----------------------------------------------------------------------------
# modules/quantize.py FAquantizer.forward_v2 (eval)
# ----------------------------------------------------------------------------
def sequence_mask(length, max_length):
    x = torch.arange(max_length, dtype=length.dtype, device=length.device)
    return x.unsqueeze(0) < length.unsqueeze(1)


def quantizer_forward(sd, x, wave, n_c=1, n_t=2, full_waves=None, wave_lens=None,
                      return_codes=False, taps=None):
    """FAquantizer.forward_v2, modules/quantize.py:375-454, eval mode (res_mask == 1)."""
    if full_waves is None:
        mel = mel_preprocess(sd, wave, n_bins=80)
        mask = torch.ones(mel.size(0), 1, mel.size(2), device=mel.device).bool()
    else:
        mel = mel_preprocess(sd, full_waves.unsqueeze(1), n_bins=80)
        mask = sequence_mask(wave_lens // HOP, mel.size(-1)).unsqueeze(1)
    timbre = style_encoder(sd, mel, mask)
    prosody_feature = mel_preprocess(sd, wave, n_bins=20)
    f0 = sconv1d(prosody_feature, sd, "melspec_linear.conv.conv")
    f0 = wavenet(sd, f0)
    f0 = sconv1d(f0, sd, "melspec_linear2.conv.conv")
    common = min(f0.size(2), x.size(2))
    f0 = f0[:, :, :common]
    x = x[:, :, :common]
    if taps is not None:
        taps["mel80"] = mel
        taps["f0_input"] = f0
    z_p, codes_p, _, cl_p, cbl_p = residual_vq(sd, "prosody_quantizer", f0, 1)
    outs = 0 + z_p
    z_c, codes_c, _, cl_c, cbl_c = residual_vq(sd, "content_quantizer", x, n_c)
    outs = outs + z_c
    residual_feature = x - z_p - z_c
    z_r, codes_r, _, cl_r, cbl_r = residual_vq(sd, "residual_quantizer", residual_feature, 3)
    outs = outs + z_r * torch.ones(z_r.shape[0], 1, 1, device=z_r.device)
    quantized = [z_p, z_c, z_r]
    codes = [codes_p, codes_c, codes_r]
    commitment = cl_p + cl_c + cl_r
    codebook = cbl_p + cbl_c + cbl_r
    style = F.linear(timbre, sd["timbre_linear.weight"], sd["timbre_linear.bias"]).unsqueeze(2)
    gamma, beta = style.chunk(2, 1)
    o = outs.transpose(1, 2)
    o = F.layer_norm(o, (o.shape[-1],), None, None, 1e-5)
    o = o.transpose(1, 2)
    o = o * gamma + beta
    if return_codes:
        return o, quantized, commitment, codebook, timbre, codes
    return o, quantized, commitment, codebook, timbre


def codec_forward(sds, wave, n_c=2):
    """reconstruct.py:56-61: encoder -> quantizer(n_c=2) -> decoder."""
    with torch.no_grad():
        z = encoder_forward(sds["encoder"], wave)
        q = quantizer_forward(sds["quantizer"], z, wave, n_c=n_c, return_codes=True)
        y = decoder_forward(sds["decoder"], q[0])
    return z, q, y


# ----------------------------------------------------------------------------
# quantize/fvq.py + quantize/rvq.py (dead code in the reference; BASELINE configs[3])
# ----------------------------------------------------------------------------
def fvq_residual_vq(layers, x, n_quantizers=None):
    """ResidualVQ.forward (eval) quantize/rvq.py:27-75 over FactorizedVectorQuantize.forward
    quantize/fvq.py:35-83.  ``layers`` = list of dicts with in_w [8,D], in_b, out_w [D,8], out_b
    (already weight-normed: weight_norm(nn.Linear) dim=0), codebook [N,8].
    Returns (quantized_out [B,D,T], indices [N,B,T], losses [N], all_quantized [N,B,D,T])."""
    quantized_out = 0.0
    residual = x
    all_idx, all_q, all_loss = [], [], []
    n = len(layers) if n_quantizers is None else n_quantizers
    for li, L in enumerate(layers):
        if li >= n:
            break
        z = residual.permute(0, 2, 1)
        z_e = F.linear(z, L["in_w"], L["in_b"]).permute(0, 2, 1)
        z_q, idx = vq_decode_latents(z_e, L["codebook"])
        z_q = z_e + (z_q - z_e)
        q = F.linear(z_q.permute(0, 2, 1), L["out_w"], L["out_b"]).permute(0, 2, 1)
        residual = residual - q
        quantized_out = quantized_out + q * 1.0
        all_idx.append(idx)
        all_q.append(q)
        all_loss.append(torch.zeros(x.shape[0]).mean())
    return quantized_out, torch.stack(all_idx), torch.stack(all_loss), torch.stack(all_q)


# ----------------------------------------------------------------------------
# alias_free_torch/ (predictor heads only; north_star asks for a kernel + parity)
# ----------------------------------------------------------------------------
def kaiser_sinc_filter1d(cutoff, half_width, kernel_size):
    """alias_free_torch/filter.py:27-58."""
    even = kernel_size % 2 == 0
    half_size = kernel_size // 2
    delta_f = 4 * half_width
    A = 2.285 * (half_size - 1) * math.pi * delta_f + 7.95
    if A > 50.0:
        beta = 0.1102 * (A - 8.7)
    elif A >= 21.0:
        beta = 0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0)
    else:
        beta = 0.0
    window = torch.kaiser_window(kernel_size, beta=beta, periodic=False)
    if even:
        time = torch.arange(-half_size, half_size) + 0.5
    else:
        time = torch.arange(kernel_size) - half_size
    filter_ = 2 * cutoff * window * torch.sinc(2 * cutoff * time)
    filter_ /= filter_.sum()
    return filter_.view(1, 1, kernel_size)


def alias_free_act(x, act, ratio=2, kernel_size=12):
    """Activation1d.forward, alias_free_torch/act.py:24-29 = UpSample1d (resample.py:28-37) ->
    act -> DownSample1d/LowPassFilter1d (resample.py:54-57, filter.py:88-96)."""
    C = x.shape[1]
    filt = kaiser_sinc_filter1d(0.5 / ratio, 0.6 / ratio, kernel_size)
    pad = kernel_size // ratio - 1
    pad_left = pad * ratio + (kernel_size - ratio) // 2
    pad_right = pad * ratio + (kernel_size - ratio + 1) // 2
    u = F.pad(x, (pad, pad), mode="replicate")
    u = ratio * F.conv_transpose1d(u, filt.expand(C, -1, -1), stride=ratio, groups=C)
    u = u[..., pad_left:-pad_right]
    u = act(u)
    even = kernel_size % 2 == 0
    pl = kernel_size // 2 - int(even)
    pr = kernel_size // 2
    d = F.pad(u, (pl, pr), mode="replicate")
    return F.conv1d(d, filt.expand(C, -1, -1), stride=ratio, groups=C)


# ----------------------------------------------------------------------------
# modules/redecoder.py (voice conversion: reconstruct_redecoder.py:108-122), encoder_type == "wavenet"
# ----------------------------------------------------------------------------
def redecoder_forward(sd, p_code, c_code, timbre_vec, use_p_code=True, use_c_code=True, n_c=2, embed_dim=512,
                      n_p_codebooks=1, causal=False):
    """Redecoder.forward, modules/redecoder.py:35-48: sum of code embeddings -> WN(hidden 512, kernel 5, 16 layers,
    gin 1024, causal = args.decoder_causal) conditioned on the timbre vector -> Conv1d(512, 1024, 1).
    p_code [B, n_p, T], c_code [B, >= n_c, T] int64, timbre_vec [B, 1024] -> [B, 1024, T]."""
    B, _, T = p_code.shape
    p_embed = torch.zeros(B, T, embed_dim)
    c_embed = torch.zeros(B, T, embed_dim)
    if use_p_code:
        for i in range(n_p_codebooks):
            p_embed += F.embedding(p_code[:, i, :], sd[f"prosody_embed.{i}.weight"])
    if use_c_code:
        for i in range(n_c):
            c_embed += F.embedding(c_code[:, i, :], sd[f"content_embed.{i}.weight"])
    x = p_embed + c_embed
    x = wavenet(sd, x.transpose(1, 2), prefix="encoder", hidden=embed_dim, n_layers=16, g=timbre_vec.unsqueeze(2),
                causal=causal) * torch.ones(B, 1, T)
    return F.conv1d(x, sd["conv_out.weight"], sd["conv_out.bias"])


def voice_convert(sds_re, codes, timbre):
    """reconstruct_redecoder.py:118-121: z = model.encoder(codes[0], codes[1], timbre, use_p_code=False, n_c=1);
    wave = model.decoder(z) with the redecoder's own non-causal, LSTM-free decoder."""
    with torch.no_grad():
        z = redecoder_forward(sds_re["encoder"], codes[0], codes[1], timbre, use_p_code=False, n_c=1)
        y = decoder_forward(sds_re["decoder"], z, causal=False, lstm=0)
    return z, y


# ----------------------------------------------------------------------------
# modules/quantize.py:29-125 predictor heads (training-only in the reference; SURVEY.md 8f rank 1)
# ----------------------------------------------------------------------------
def snake_beta(x, alpha, beta, alpha_logscale=True):
    """SnakeBeta.forward, modules/quantize.py:78-88."""
    a = alpha.unsqueeze(0).unsqueeze(-1)
    b = beta.unsqueeze(0).unsqueeze(-1)
    if alpha_logscale:
        a = torch.exp(a)
        b = torch.exp(b)
    return x + (1.0 / (b + 0.000000001)) * torch.pow(torch.sin(x * a), 2)


def _head_act(x, sd, prefix):
    """Activation1d(activation=SnakeBeta(dim, alpha_logscale=True)), modules/quantize.py:97."""
    return alias_free_act(x, lambda u: snake_beta(u, sd[prefix + ".act.alpha"], sd[prefix + ".act.beta"]))


def head_residual_unit(x, sd, prefix, dilation):
    """modules/quantize.py:90-104 ResidualUnit: plain weight-normed nn.Conv1d (zero padding ((7-1)*d)//2), NOT SConv1d."""
    y = _head_act(x, sd, prefix + ".block.0")
    y = F.conv1d(y, _wn_weight(sd, prefix + ".block.1"), sd[prefix + ".block.1.bias"], dilation=dilation,
                 padding=((7 - 1) * dilation) // 2)
    y = _head_act(y, sd, prefix + ".block.2")
    y = F.conv1d(y, _wn_weight(sd, prefix + ".block.3"), sd[prefix + ".block.3.bias"])
    return x + y


def cnnlstm_forward(sd, x, n_heads, global_pred=False):
    """CNNLSTM.forward, modules/quantize.py:106-125 (despite the name: 3 ResidualUnits (dilation 1, 2, 3), an alias-free
    SnakeBeta, then ``n_heads`` nn.Linear heads; no LSTM in the reference class).  x [B, C, T] -> list of [B, T, out]
    (or [B, out] when global_pred)."""
    h = x
    for j, d in enumerate((1, 2, 3)):
        h = head_residual_unit(h, sd, f"model.{j}", d)
    h = _head_act(h, sd, "model.3")
    h = h.transpose(1, 2)
    if global_pred:
        h = torch.mean(h, dim=1, keepdim=False)
    return [F.linear(h, sd[f"heads.{i}.weight"], sd[f"heads.{i}.bias"]) for i in range(n_heads)]


def fa_predictors_forward(sd, quantized, timbre=None, use_gr_content_f0=False, use_gr_prosody_phone=False,
                          use_gr_residual_f0=False, use_gr_residual_phone=False, use_gr_timbre_content=True,
                          use_gr_timbre_prosody=True, use_gr_x_timbre=False, norm_f0=True, timbre_norm=False):
    """FApredictors.forward (modules/quantize.py:507-563) / forward_v2 (:564-619, when timbre_norm) over the module's
    state_dict: the GradientReversal layers are identities in the forward pass; the reversal heads sit at index 1 of their
    nn.Sequential (keys ``rev_*_predictor.1.*``)."""
    sub = lambda name: {k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")}
    head = lambda name, x, n, glob=False: cnnlstm_forward(sub(name), x, n, global_pred=glob)
    if timbre_norm:
        p, c, r = quantized[0], quantized[1], quantized[2]
        content_pred = head("phone_predictor", c, 1)[0]
        spk_pred = F.linear(timbre, sd["timbre_predictor.weight"], sd["timbre_predictor.bias"])
        f0_pred, uv_pred = head("f0_predictor", p, 2)
        prosody_rev = torch.zeros_like(p)
        if use_gr_content_f0:
            prosody_rev = prosody_rev + c
        if use_gr_residual_f0:
            prosody_rev = prosody_rev + r
        rev_f0_pred, rev_uv_pred = head("rev_f0_predictor.1", prosody_rev, 2)
        content_rev = torch.zeros_like(c)
        if use_gr_prosody_phone:
            content_rev = content_rev + p
        if use_gr_residual_phone:
            content_rev = content_rev + r
        rev_content_pred = head("rev_content_predictor.1", content_rev, 1)[0]
        timbre_rev = p + c + r
    else:
        p, c, t, r = quantized[0], quantized[1], quantized[2], quantized[3]
        content_pred = head("phone_predictor", c, 1)[0]
        if norm_f0:
            spk_pred = head("timbre_predictor", t, 1, True)[0]
            f0_pred, uv_pred = head("f0_predictor", p, 2)
        else:
            spk_pred = head("timbre_predictor", t + p, 1, True)[0]
            f0_pred, uv_pred = head("f0_predictor", p + t, 2)
        prosody_rev = torch.zeros_like(p)
        for flag, lat in ((use_gr_content_f0, c), (use_gr_timbre_prosody, t), (use_gr_residual_f0, r)):
            if flag:
                prosody_rev = prosody_rev + lat
        rev_f0_pred, rev_uv_pred = head("rev_f0_predictor.1", prosody_rev, 2)
        content_rev = torch.zeros_like(c)
        for flag, lat in ((use_gr_prosody_phone, p), (use_gr_timbre_content, t), (use_gr_residual_phone, r)):
            if flag:
                content_rev = content_rev + lat
        rev_content_pred = head("rev_content_predictor.1", content_rev, 1)[0]
        timbre_rev = p + c + r if norm_f0 else c + r
    x_spk_pred = head("rev_timbre_predictor.1", timbre_rev, 1, True)[0] if use_gr_x_timbre else None
    preds = {"f0": f0_pred, "uv": uv_pred, "content": content_pred, "timbre": spk_pred}
    rev_preds = {"rev_f0": rev_f0_pred, "rev_uv": rev_uv_pred, "rev_content": rev_content_pred, "x_timbre": x_spk_pred}
    return preds, rev_preds


# ----------------------------------------------------------------------------
# meldataset.py:29-47 dataset-side mel (PseudoDataset training targets)
# ----------------------------------------------------------------------------
def dataset_mel(wave, window, fb, n_fft=2048, hop=HOP, win_length=1200):
    """meldataset.py:37-47 preprocess: to_mel = torchaudio MelSpectrogram(n_mels=80, n_fft=2048, win_length=1200,
    hop_length=300) with its DEFAULT sample_rate=16000 (the filterbank differs from the quantizer's 24 kHz one),
    then (log(1e-5 + mel) + 4) / 4.  wave [T] or [B, T] -> [B, 80, T // 300 + 1] (no frame slicing here)."""
    if wave.dim() == 1:
        wave = wave.unsqueeze(0)
    spec = torch.stft(wave, n_fft, hop_length=hop, win_length=win_length, window=window, center=True, pad_mode="reflect",
                      normalized=False, onesided=True, return_complex=True)
    spec = spec.abs().pow(2.0)
    mel = torch.matmul(spec.transpose(-1, -2), fb).transpose(-1, -2)
    return (torch.log(1e-5 + mel) - (-4)) / 4


# ----------------------------------------------------------------------------
# losses.py:65-89 reconstruction_loss (training-side loss forward)
# ----------------------------------------------------------------------------
def reconstruction_loss(x, G_x, eps=1e-7, return_terms=False):
    """losses.py:65-89: 100 * mse + sum_{i=6..11} (l1 + sqrt(2^i / 2) * l2) over torchaudio MelSpectrogram(sample_rate=16000,
    n_fft=max(s, 512), win_length=s, hop_length=s // 4, n_mels=64), restated with torch.stft + the HTK filterbank the
    transform builds (torchaudio.functional.melscale_fbanks) -- the same ATen calls in the same order."""
    import torch.nn.functional as F
    import torchaudio
    L = 100 * F.mse_loss(x, G_x)
    terms = [F.mse_loss(x, G_x)]
    for i in range(6, 12):
        s = 2 ** i
        n_fft = max(s, 512)
        window = torch.hann_window(s, device=x.device)
        fb = torchaudio.functional.melscale_fbanks(n_fft // 2 + 1, 0.0, 8000.0, 64, 16000, None, "htk").to(x.device)

        def melspec(w):
            shape = w.shape
            spec = torch.stft(w.reshape(-1, shape[-1]), n_fft, hop_length=s // 4, win_length=s, window=window, center=True,
                              pad_mode="reflect", normalized=False, onesided=True, return_complex=True)
            spec = spec.reshape(shape[:-1] + spec.shape[-2:]).abs().pow(2.0)
            return torch.matmul(spec.transpose(-1, -2), fb).transpose(-1, -2)

        S_x, S_G_x = melspec(x), melspec(G_x)
        l1_loss = (S_x - S_G_x).abs().mean()
        l2_loss = (((torch.log(S_x.abs() + eps) - torch.log(S_G_x.abs() + eps)) ** 2).mean(dim=-2) ** 0.5).mean()
        alpha = (s / 2) ** 0.5
        L = L + (l1_loss + alpha * l2_loss)
        terms += [l1_loss, l2_loss]
    return (L, torch.stack(terms)) if return_terms else L


# ----------------------------------------------------------------------------
# dac/nn/loss.py:11-47, :142-327 L1Loss / MultiScaleSTFTLoss / MelSpectrogramLoss
# PARITY UNPINNED: the reference evaluates them on audiotools.AudioSignal (AudioSignal.stft / .magnitude / .mel_spectrogram),
# and neither audiotools nor librosa is installed or vendored (SURVEY.md 8c).  Their published semantics are restated here;
# the Slaney filterbank is cross-checked against torchaudio's own Slaney implementation (tests/test_oracle.py).
# ----------------------------------------------------------------------------
def librosa_mel_filters(sr, n_fft, n_mels, fmin=0.0, fmax=None, dtype=torch.float32):
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) with its defaults (htk=False: Slaney mel scale; norm='slaney':
    each triangle divided by half its width in Hz), evaluated in float64 and rounded to ``dtype`` (float32, as librosa
    returns it; float64 keeps the unrounded values).  Returns [n_mels, 1 + n_fft // 2]."""
    import numpy as np
    fmax = sr / 2.0 if fmax is None else float(fmax)
    f_sp, min_log_hz = 200.0 / 3.0, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    hz2mel = lambda f: np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, f / f_sp)
    mel2hz = lambda m: np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)
    fftfreqs = np.linspace(0.0, sr / 2.0, 1 + n_fft // 2)
    mel_f = mel2hz(np.linspace(hz2mel(np.float64(fmin)), hz2mel(np.float64(fmax)), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        w[i] = np.maximum(0.0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return torch.from_numpy(w).to(dtype)


def _audiotools_magnitude(x, w):
    """AudioSignal(x).stft(window_length=w, hop_length=w // 4) -> .magnitude, [B, C, w // 2 + 1, frames]."""
    shape = x.shape
    win = torch.hann_window(w, periodic=True, device=x.device)          # scipy.signal.get_window("hann", w) (fftbins=True)
    st = torch.stft(x.reshape(-1, shape[-1]), n_fft=w, hop_length=w // 4, window=win, return_complex=True, center=True)
    return st.abs().reshape(shape[:-1] + st.shape[-2:])


def multiscale_stft_loss(x, y, window_lengths=(2048, 512), clamp_eps=1e-5, mag_weight=1.0, log_weight=1.0, pow=2.0):
    """dac/nn/loss.py:201-231 with loss_fn = nn.L1Loss()."""
    loss = 0.0
    for w in window_lengths:
        mx, my = _audiotools_magnitude(x, w), _audiotools_magnitude(y, w)
        loss = loss + log_weight * F.l1_loss(mx.clamp(clamp_eps).pow(pow).log10(), my.clamp(clamp_eps).pow(pow).log10())
        loss = loss + mag_weight * F.l1_loss(mx, my)
    return loss


def mel_spectrogram_loss(x, y, sample_rate=24000, n_mels=(150, 80), window_lengths=(2048, 512), clamp_eps=1e-5, mag_weight=1.0,
                         log_weight=1.0, pow=2.0, mel_fmin=(0.0, 0.0), mel_fmax=(None, None)):
    """dac/nn/loss.py:297-327 with loss_fn = nn.L1Loss(); mel_spectrogram = (magnitude.transpose(2, -1) @ mel_basis.T).transpose(-1, 2)."""
    loss = 0.0
    for nm, f0, f1, w in zip(n_mels, mel_fmin, mel_fmax, window_lengths):
        basis = librosa_mel_filters(sample_rate, w, nm, f0, f1).to(x.device)
        mel = lambda m: (m.transpose(2, -1) @ basis.T).transpose(-1, 2)
        mx, my = mel(_audiotools_magnitude(x, w)), mel(_audiotools_magnitude(y, w))
        loss = loss + log_weight * F.l1_loss(mx.clamp(clamp_eps).pow(pow).log10(), my.clamp(clamp_eps).pow(pow).log10())
        loss = loss + mag_weight * F.l1_loss(mx, my)
    return loss
