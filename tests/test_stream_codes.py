"""Streaming compression to codes (fac_stream_encode_codes / fac_stream_finish_codes, CodecStream.encode_codes /
finish_codes): an utterance fed in chunks must give the codes and the timbre of ONE offline Codec.encode, bit for bit.

What makes that possible (include/facodec_b200.h): mel frame t covers samples [300 t - 600, 300 t + 600), so the stream holds
back one frame until the end; the prosody WaveNet (8 causal k = 5 convs, each reflect-padding 4 frames at its window's left
edge) is recomputed over <= 32 frames of mel history; the timbre pools over every mel frame, so it exists only at the end.
The schedule is pinned on the CPU oracle first, then the engine is held to bit-identity on the GPU.
"""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN_CASES, case_inputs, load_golden, state_dicts

HOP, WN_CTX, MEL_HIST = 300, 32, 900


def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    new = ("fac_stream_encode_codes", "fac_stream_finish_codes")
    assert set(new) <= set(_declared("facodec_b200.h"))
    assert set(new) <= set(_lib.EXPORTED)


def _oracle_mel80(sd, seg, n_frames):
    """mel80 rows of the centred STFT from an explicit sample segment [300 f - 600, 300 (f + n) + 600) (already reflected
    where it reaches past the utterance): 1200-sample Hann frames zero-padded to n_fft = 2048, as torch.stft pads them."""
    fr = seg.unfold(-1, 1200, HOP)[..., :n_frames, :] * sd["to_mel.spectrogram.window"]
    spec = torch.fft.rfft(F.pad(fr, (424, 424)), n=2048).abs().pow(2.0)
    mel = spec @ sd["to_mel.mel_scale.fb"]
    return ((torch.log(1e-5 + mel) + 4) / 4).transpose(-1, -2)     # [B, 80, n]


@torch.no_grad()
def test_stream_schedule_on_oracle():
    """The stream's schedule restated on the fp32 oracle (no GPU): 6000-sample chunks, mel frames cut from a 900-sample
    history (reflected only at the utterance's true start and end), one frame held back, the prosody net recomputed over
    <= 32 frames of mel history.  It reproduces the offline f0_input and, through the oracle VQ, the golden codes."""
    from oracle import facodec_oracle as O
    c = GOLDEN_CASES["b1_t96000"]
    g = load_golden("b1_t96000")
    sd = state_dicts(c["wseed"])["quantizer"]
    x, _ = case_inputs(c)
    z = torch.as_tensor(g["z"])
    T = x.shape[-1]

    def prosody(mel20):
        f0 = O.sconv1d(mel20, sd, "melspec_linear.conv.conv")
        return O.sconv1d(O.wavenet(sd, f0), sd, "melspec_linear2.conv.conv")

    mels, f0s, emitted = [], [], 0
    for p in range(0, T, 6000):
        seen = p + 6000
        last = seen // HOP - 1 if seen < T else seen // HOP      # the last frame seen waits for the end of the stream
        lo_s = max(0, p - MEL_HIST)                              # what the stream still holds of the past samples
        idx = torch.arange(emitted * HOP - 600, (last - 1) * HOP + 600)
        idx = torch.where(idx < 0, -idx, idx)                    # reflect at the true start
        if seen >= T:
            idx = torch.where(idx >= T, 2 * (T - 1) - idx, idx)  # ... and at the true end
        assert int(idx.min()) >= lo_s and int(idx.max()) < seen
        mels.append(_oracle_mel80(sd, x[:, 0, idx], last - emitted))
        allm = torch.cat(mels, dim=2)
        lo = max(0, emitted - WN_CTX)
        f0s.append(prosody(allm[:, :20, lo:last])[:, :, emitted - lo:])
        emitted = last
    assert emitted == T // HOP
    f0_st = torch.cat(f0s, dim=2)
    f0_off = prosody(O.mel_preprocess(sd, x, n_bins=80)[:, :20])
    assert float((f0_st - f0_off).abs().max()) <= 1e-5
    zp, cp, *_ = O.residual_vq(sd, "prosody_quantizer", f0_st, 1)
    zc, cc, *_ = O.residual_vq(sd, "content_quantizer", z, 2)
    _, cr, *_ = O.residual_vq(sd, "residual_quantizer", z - zp - zc, 3)
    for k, v in zip(("codes_p", "codes_c", "codes_r"), (cp, cc, cr)):
        assert np.array_equal(v.numpy(), g[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _stream_codes(s, x, sizes, n_c):
    from test_gpu_stream import chunks_of
    parts = [s.encode_codes(x[:, :, p:p + n].contiguous(), n_c) for p, n in chunks_of(x.shape[-1], sizes)]
    last, timbre = s.finish_codes()
    codes = [torch.cat([q[i] for q in parts] + [last[i]], dim=2) for i in range(3)]
    return codes, timbre, parts


def _waves(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 1, T, generator=g) * 0.1).to("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("n_c", [1, 2])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("sizes", [[3000, 300, 9000, 24000, 600], [30000], [4500, 1500]])
def test_stream_codes_equal_offline(sizes, B, n_c, built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    m = model_for(1)
    x = _waves(B, 60000, 77 + B)
    codes_off, timbre_off = fb.Codec(m).encode(x, n_c)
    with fb.CodecStream(m, B) as s:
        codes, timbre, parts = _stream_codes(s, x, sizes, n_c)
    torch.cuda.synchronize()
    from test_gpu_stream import chunks_of
    assert [q[0].shape[2] for q in parts] == [n // HOP - (p == 0) for p, n in chunks_of(60000, sizes)]
    for k, a, b in zip(("codes_p", "codes_c", "codes_r"), codes, codes_off):
        assert a.shape == b.shape and torch.equal(a, b), k
    assert torch.equal(timbre, timbre_off)


@pytest.mark.gpu
@pytest.mark.parametrize("name,sizes", [("b1_t96000", [6000]), ("b2_t7200", [3000, 4200])])
def test_stream_codes_golden(name, sizes, built_lib):
    """The reference's own codes (golden fixtures made from the imported reference)."""
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    c = GOLDEN_CASES[name]
    gold = load_golden(name)
    m = model_for(c["wseed"])
    x, _ = case_inputs(c)
    with fb.CodecStream(m, c["B"]) as s:
        codes, _, _ = _stream_codes(s, x.to("cuda:0"), sizes, c["n_c"])
    for k, cg in zip(("codes_p", "codes_c", "codes_r"), codes):
        assert np.array_equal(cg.cpu().numpy(), gold[k]), k


@pytest.mark.gpu
def test_live_sender_receiver(built_lib):
    """One stream compresses chunks as they arrive and decodes the codes as they come out (buffered only until the
    decoder's first 10 frames exist), with the timbre of the whole utterance: the waveform of Codec.decode."""
    import facodec_b200 as fb
    from test_gpu_parity import RMS_TOL, model_for, rms
    from test_gpu_stream import chunks_of
    m = model_for(1)
    x = _waves(1, 48000, 5)
    codec = fb.Codec(m)
    codes_off, timbre = codec.encode(x, 2)
    y_off = codec.decode(codes_off, timbre)
    ys, pending = [], []

    def feed(codes, final=False):
        pending.append(codes)
        if ys or final or sum(q[0].shape[2] for q in pending) >= 10:
            ys.append(s.decode_codes([torch.cat([q[i] for q in pending], dim=2) for i in range(3)], timbre))
            pending.clear()

    with fb.CodecStream(m, 1) as s:
        for p, n in chunks_of(x.shape[-1], [3000, 6000]):
            feed(s.encode_codes(x[:, :, p:p + n].contiguous(), 2))
        feed(s.finish_codes()[0], final=True)
    y = torch.cat(ys, dim=2)
    torch.cuda.synchronize()
    assert y.shape == y_off.shape
    assert rms(y, y_off) <= RMS_TOL
    print("live stream vs Codec.decode: rms %.3g bit-equal %s" % (rms(y, y_off), bool(torch.equal(y, y_off))))


@pytest.mark.gpu
def test_two_streams_interleaved(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    from test_gpu_stream import chunks_of
    m = model_for(1)
    xa, xb = _waves(2, 36000, 11), _waves(2, 36000, 12)
    codec = fb.Codec(m)
    off = [codec.encode(xa, 2), codec.encode(xb, 2)]
    with fb.CodecStream(m, 2) as sa, fb.CodecStream(m, 2) as sb:
        got = [[], []]
        for ca, cb in itertools.zip_longest(chunks_of(36000, [6000, 3000]), chunks_of(36000, [3300, 6600, 2100])):
            for j, s, x, ch in ((0, sa, xa, ca), (1, sb, xb, cb)):
                if ch is not None:
                    got[j].append(s.encode_codes(x[:, :, ch[0]:ch[0] + ch[1]].contiguous(), 2))
        fins = [sa.finish_codes(), sb.finish_codes()]
    for j in range(2):
        codes = [torch.cat([q[i] for q in got[j]] + [fins[j][0][i]], dim=2) for i in range(3)]
        for a, b in zip(codes, off[j][0]):
            assert torch.equal(a, b)
        assert torch.equal(fins[j][1], off[j][1])


@pytest.mark.gpu
def test_stream_codes_error_paths(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    m = model_for(1)
    dev = torch.device("cuda:0")
    x = _waves(1, 12000, 3)
    with fb.CodecStream(m, 1) as s:
        with pytest.raises(fb.FacError):
            s.finish_codes()                                     # nothing encoded
        with pytest.raises(fb.FacError):
            s.encode_codes(torch.zeros(1, 1, 2700, device=dev))  # first chunk < 3000
        with pytest.raises(fb.FacError):
            s.encode_codes(torch.zeros(1, 1, 3100, device=dev))  # not a multiple of 300
        with pytest.raises(fb.FacError):
            s.encode_codes(torch.zeros(1, 1, 3000))              # CPU tensor
        got = [s.encode_codes(x[:, :, :3000].contiguous(), 2)]
        with pytest.raises(fb.FacError):
            s.encode_codes(x[:, :, 3000:6000].contiguous(), 1)   # n_c changed mid-stream
        with pytest.raises(fb.FacError):
            s.encode(x[:, :, 3000:6000].contiguous())            # latents on a codes stream
        # the rejected calls left the stream as it was
        got.append(s.encode_codes(x[:, :, 3000:].contiguous(), 2))
        last, timbre = s.finish_codes()
        with pytest.raises(fb.FacError):
            s.encode_codes(x[:, :, :3000].contiguous(), 2)       # after finish_codes
        with pytest.raises(fb.FacError):
            s.finish_codes()
    codes_off, timbre_off = fb.Codec(m).encode(x, 2)
    for i in range(3):
        assert torch.equal(torch.cat([got[0][i], got[1][i], last[i]], dim=2), codes_off[i])
    assert torch.equal(timbre, timbre_off)
    with fb.CodecStream(m, 1) as s:
        s.encode(x[:, :, :3000].contiguous())
        with pytest.raises(fb.FacError):
            s.encode_codes(x[:, :, 3000:6000].contiguous())      # codes on a latents stream
    try:
        m.encoder._engine.set_option("tensor_cores", 1)
        with fb.CodecStream(m, 1) as s:
            with pytest.raises(fb.FacError):
                s.encode_codes(x[:, :, :3000].contiguous())
    finally:
        m.encoder._engine.set_option("tensor_cores", 2)
