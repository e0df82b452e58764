"""Streaming voice conversion through the redecoder (fac_vc_stream_*, VoiceConversionStream): codes fed in chunks must give
the waveform of ONE offline VoiceConverter.convert on the whole utterance, bit for bit.

The redecoder (16 WN layers of non-causal k = 5 convs) and its decoder (centred k = 7 convs, 3-tap transposed convs) are
non-causal but hold no LSTM: z frame t reads codes [t - 32, t + 32] and output frame t reads z frames [t - 12, t + 12], so
output frame t is final once code frame t + 44 has arrived.  Windows carry that much context on both sides and reflect only
at the utterance's true start and end.  The reach is pinned on the fp64 oracle, the schedule on the fp32 oracle, and then the
engine is held to bit-identity on the GPU.
"""
import itertools

import pytest
import torch

from conftest import REDEC_CASES, load_golden

HOP, RED_CTX, DEC_CTX = 300, 32, 12
CHUNKINGS = {"ones": [1], "twenty": [20], "mixed": [7, 1, 50, 13], "one_call": [100000]}


def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    new = ("fac_vc_stream_lookahead", "fac_vc_stream_begin", "fac_vc_stream_convert", "fac_vc_stream_finish", "fac_vc_stream_end")
    assert set(new) <= set(_declared("facodec_b200.h"))
    assert set(new) <= set(_lib.EXPORTED)


def _sds64(seed):
    from facodec_b200 import synth
    return {k: {n: v.double() if v.is_floating_point() else v for n, v in sd.items()}
            for k, sd in synth.synth_redecoder_state_dicts(seed).items()}


def _codes(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(0, 1024, (B, 1, T), generator=g), torch.randint(0, 1024, (B, 2, T), generator=g),
            torch.randn(B, 1024, generator=g))


def _changed(a, b):
    d = torch.nonzero((a - b).abs().reshape(-1, a.shape[-1]).amax(dim=0)).view(-1)
    return int(d.min()), int(d.max())


@torch.no_grad()
def test_reach_pin_on_oracle(built_lib):
    """fp64 oracle perturbations: one code changes exactly z frames [t - 32, t + 32]; one z frame f changes exactly output
    samples [300 f - 3547, 300 f + 3834], i.e. output frame t reads z frames [t - 12, t + 12].  fac_vc_stream_lookahead()
    is their sum (host-only call)."""
    from facodec_b200 import _lib
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)          # the oracle's embedding sums start from default-dtype zeros
    try:
        lo, hi = _reach_fp64()
    finally:
        torch.set_default_dtype(prev)
    assert (lo, hi) == (-3547, 3834)
    ahead, behind = (HOP - 1 - lo) // HOP, hi // HOP      # z frames after / before output frame t that it reads
    assert ahead == behind == DEC_CTX
    assert _lib.load().fac_vc_stream_lookahead() == RED_CTX + DEC_CTX == 44


def _reach_fp64():
    from oracle import facodec_oracle as O
    sds = _sds64(0)
    cp, cc, tv = _codes(1, 100, 3)
    tv = tv.double()
    z = O.redecoder_forward(sds["encoder"], cp, cc, tv, use_p_code=True, n_c=2)
    t = 50
    for row in range(3):
        p2, c2 = cp.clone(), cc.clone()
        v = p2[0, 0] if row == 0 else c2[0, row - 1]
        v[t] = (v[t] + 1) % 1024
        z2 = O.redecoder_forward(sds["encoder"], p2, c2, tv, use_p_code=True, n_c=2)
        assert _changed(z, z2) == (t - RED_CTX, t + RED_CTX), row
    zs = z[:, :, :30]
    f = 15
    y = O.decoder_forward(sds["decoder"], zs, causal=False, lstm=0)
    zp = zs.clone()
    zp[:, :, f] += 1.0
    lo, hi = _changed(y, O.decoder_forward(sds["decoder"], zp, causal=False, lstm=0))
    return lo - HOP * f, hi - HOP * f


def _frame_counts(sizes, T):
    """Frames each convert() returns, then finish(): output frame t is emitted once code frame t + 44 is in."""
    from test_gpu_stream import chunks_of
    out, prev = [], 0
    for p, n in chunks_of(T, sizes):
        out.append(max(0, p + n - RED_CTX - DEC_CTX) - prev)
        prev += out[-1]
    return out + [T - prev]


@torch.no_grad()
def _oracle_stream(sds, cp, cc, tv, sizes, use_p, n_c, red_ctx=RED_CTX, dec_ctx=DEC_CTX):
    """The engine's schedule on the oracle: after N code frames, z frames [Zf, N - red_ctx) come from the redecoder over
    codes [max(0, Zf - red_ctx), N), and output frames [Yf, Zf - dec_ctx) from the decoder over z [max(0, Yf - dec_ctx), Zf);
    only those clean rows are kept.  finish() runs both to the true end."""
    from oracle import facodec_oracle as O
    from test_gpu_stream import chunks_of
    T = cp.shape[-1]
    z = torch.zeros(cp.shape[0], 1024, 0, dtype=tv.dtype)
    ys, st = [], dict(Zf=0, Yf=0)

    def step(N, Zf1, Yf1):
        Zf, Yf = st["Zf"], st["Yf"]
        nonlocal z
        if Zf1 > Zf:
            lo = max(0, Zf - red_ctx)
            zw = O.redecoder_forward(sds["encoder"], cp[:, :, lo:N], cc[:, :, lo:N], tv, use_p_code=use_p, n_c=n_c)
            z = torch.cat([z, zw[:, :, Zf - lo:Zf1 - lo]], dim=2)
        if Yf1 > Yf:
            lo = max(0, Yf - dec_ctx)
            yw = O.decoder_forward(sds["decoder"], z[:, :, lo:Zf1], causal=False, lstm=0)
            ys.append(yw[:, :, (Yf - lo) * HOP:(Yf1 - lo) * HOP])
        st.update(Zf=Zf1, Yf=Yf1)

    for p, n in chunks_of(T, sizes):
        Zf1 = max(st["Zf"], p + n - red_ctx)
        step(p + n, Zf1, max(st["Yf"], Zf1 - dec_ctx))
    step(T, T, T)
    return torch.cat(ys, dim=2)


@pytest.mark.parametrize("T,sizes", [(150, "ones"), (150, "twenty"), (150, "mixed"), (150, "one_call"), (5, "twenty"),
                                     (5, "ones")])
def test_stream_schedule_on_oracle(T, sizes):
    """The schedule restated on the fp32 oracle reproduces O.voice_convert within fp32 rounding (1e-5 of the peak)."""
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    sds = synth.synth_redecoder_state_dicts(0)
    cp, cc, tv = _codes(1, T, 11)
    _, y_off = O.voice_convert(sds, [cp, cc], tv)
    y = _oracle_stream(sds, cp, cc, tv, CHUNKINGS[sizes], use_p=False, n_c=1)
    assert y.shape == y_off.shape
    assert float((y - y_off).abs().max()) <= 1e-5 * float(y_off.abs().max())


def test_stream_schedule_exact_in_fp64():
    """On the fp64 oracle the schedule reproduces the offline call to fp64 rounding (<= 1e-13 of the peak), and with one
    frame less of decoder context it does not (measured 3.4e-6 of the peak: a window edge reaches a kept output frame
    through the decoder's far taps, below what the fp32 bar above can see).  One frame less of redecoder context stays at
    fp64 rounding (measured 1.9e-15): that corruption crosses 16 chained edge taps of the WN and vanishes, so only the
    perturbation pin above shows the 32."""
    from oracle import facodec_oracle as O
    sds = _sds64(0)
    cp, cc, tv = _codes(1, 90, 12)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        tv = tv.double()
        _, y_off = O.voice_convert(sds, [cp, cc], tv)
        err = {}
        for ctx in ((RED_CTX, DEC_CTX), (RED_CTX, DEC_CTX - 1)):
            y = _oracle_stream(sds, cp, cc, tv, [20], use_p=False, n_c=1, red_ctx=ctx[0], dec_ctx=ctx[1])
            err[ctx] = float((y - y_off).abs().max()) / float(y_off.abs().max())
    finally:
        torch.set_default_dtype(prev)
    assert err[(RED_CTX, DEC_CTX)] <= 1e-13, err
    assert err[(RED_CTX, DEC_CTX - 1)] > 1e-8, err


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _dev_codes(B, T, seed):
    return tuple(t.to("cuda:0") for t in _codes(B, T, seed))


def _stream_convert(s, cp, cc, sizes):
    """convert() on each chunk, then finish(): the list of outputs."""
    from test_gpu_stream import chunks_of
    ys = [s.convert([cp[:, :, p:p + n], cc[:, :, p:p + n]]) for p, n in chunks_of(cp.shape[-1], sizes)]
    return ys + [s.finish()]


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", list(CHUNKINGS))
@pytest.mark.parametrize("T", [5, 44, 45, 300])
@pytest.mark.parametrize("use_p,n_c", [(False, 1), (True, 2)])
@pytest.mark.parametrize("B", [1, 3])
def test_vc_stream_equal_offline(B, use_p, n_c, T, sizes, built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    cp, cc, tv = _dev_codes(B, T, 100 + T + B)
    y_off = fb.VoiceConverter(m).convert([cp, cc], tv, use_p_code=use_p, n_c=n_c)
    with fb.VoiceConversionStream(m, B, tv, use_p_code=use_p, n_c=n_c) as s:
        assert s.lookahead_frames == RED_CTX + DEC_CTX
        ys = _stream_convert(s, cp, cc, CHUNKINGS[sizes])
    torch.cuda.synchronize()
    assert [y.shape[2] // HOP for y in ys] == _frame_counts(CHUNKINGS[sizes], T)
    y = torch.cat(ys, dim=2)
    assert y.shape == y_off.shape and torch.equal(y, y_off)


@pytest.mark.gpu
@pytest.mark.parametrize("name,sizes", [("redec_b2_t7200_vc", "mixed"), ("redec_b2_t7200_vc", "ones"),
                                        ("redec_b3_t1500_short", "ones")])
def test_vc_stream_golden(name, sizes, built_lib):
    """The reference's own voice-conversion output (golden fixtures made from the imported reference), fed in chunks."""
    import facodec_b200 as fb
    from test_gpu_parity import RMS_TOL, redec_model_for, rms
    c = REDEC_CASES[name]
    g = load_golden(name)
    src = load_golden(c["src"])
    m = redec_model_for(c["wseed"])
    cp, cc, tv = (torch.from_numpy(src[k]).to("cuda:0") for k in ("codes_p", "codes_c", "timbre"))
    y_off = fb.VoiceConverter(m).convert([cp, cc], tv, use_p_code=c["use_p"], n_c=c["n_c"])
    with fb.VoiceConversionStream(m, cp.shape[0], tv, use_p_code=c["use_p"], n_c=c["n_c"]) as s:
        y = torch.cat(_stream_convert(s, cp, cc, CHUNKINGS[sizes]), dim=2)
    torch.cuda.synchronize()
    assert torch.equal(y, y_off)
    assert rms(y, g["y"]) <= RMS_TOL


@pytest.mark.gpu
def test_live_voice_conversion_pipeline(built_lib):
    """reconstruct_redecoder.py:118-121 live: a source signal is compressed chunk by chunk (CodecStream.encode_codes) and
    its codes go straight into a VoiceConversionStream holding the timbre of Codec.encode(reference)."""
    import facodec_b200 as fb
    from facodec_b200 import synth
    from test_gpu_parity import model_for, redec_model_for
    from test_gpu_stream import chunks_of
    codec, rm = model_for(0), redec_model_for(0)
    src = synth.synth_waves(1, 36000, seed=41).to("cuda:0")
    ref = synth.synth_waves(1, 12000, seed=42).to("cuda:0")
    _, timbre = fb.Codec(codec).encode(ref, 2)
    codes_off, _ = fb.Codec(codec).encode(src, 2)
    y_off = fb.VoiceConverter(rm).convert(codes_off, timbre, use_p_code=False, n_c=1)
    ys = []
    with fb.CodecStream(codec, 1) as tx, fb.VoiceConversionStream(rm, 1, timbre, use_p_code=False, n_c=1) as vc:
        for p, n in chunks_of(src.shape[-1], [3000, 300, 6000]):
            ys.append(vc.convert(tx.encode_codes(src[:, :, p:p + n].contiguous(), 2)))
        ys.append(vc.convert(tx.finish_codes()[0]))
        ys.append(vc.finish())
    y = torch.cat(ys, dim=2)
    torch.cuda.synchronize()
    assert y.shape == y_off.shape and torch.equal(y, y_off)


@pytest.mark.gpu
def test_vc_streams_interleaved_beside_codec_stream(built_lib):
    """Two VC streams on the redecoder's handle, interleaved call by call with a CodecStream on the codec's handle."""
    import facodec_b200 as fb
    from facodec_b200 import synth
    from test_gpu_parity import model_for, redec_model_for
    from test_gpu_stream import chunks_of
    codec, rm = model_for(0), redec_model_for(0)
    vc = fb.VoiceConverter(rm)
    a, b = _dev_codes(2, 120, 1), _dev_codes(3, 97, 2)
    off_a = vc.convert(a[:2], a[2])
    off_b = vc.convert(b[:2], b[2], use_p_code=True, n_c=2)
    x = synth.synth_waves(1, 36000, seed=43).to("cuda:0")
    codes_off, timbre_off = fb.Codec(codec).encode(x, 2)
    got = [[], [], []]
    with fb.VoiceConversionStream(rm, 2, a[2]) as sa, fb.VoiceConversionStream(rm, 3, b[2], use_p_code=True, n_c=2) as sb, \
            fb.CodecStream(codec, 1) as tx:
        for ca, cb, cx in itertools.zip_longest(chunks_of(120, [20]), chunks_of(97, [7, 1, 50, 13]), chunks_of(36000, [6000])):
            if ca is not None:
                got[0].append(sa.convert([a[0][:, :, ca[0]:ca[0] + ca[1]], a[1][:, :, ca[0]:ca[0] + ca[1]]]))
            if cb is not None:
                got[1].append(sb.convert([b[0][:, :, cb[0]:cb[0] + cb[1]], b[1][:, :, cb[0]:cb[0] + cb[1]]]))
            if cx is not None:
                got[2].append(tx.encode_codes(x[:, :, cx[0]:cx[0] + cx[1]].contiguous(), 2))
        got[0].append(sa.finish())
        got[1].append(sb.finish())
        last, timbre = tx.finish_codes()
    assert torch.equal(torch.cat(got[0], dim=2), off_a)
    assert torch.equal(torch.cat(got[1], dim=2), off_b)
    for i in range(3):
        assert torch.equal(torch.cat([q[i] for q in got[2]] + [last[i]], dim=2), codes_off[i])
    assert torch.equal(timbre, timbre_off)


@pytest.mark.gpu
def test_vc_stream_batch_32(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    cp, cc, tv = _dev_codes(32, 160, 5)
    y_off = fb.VoiceConverter(m).convert([cp, cc], tv)
    with fb.VoiceConversionStream(m, 32, tv) as s:
        y = torch.cat(_stream_convert(s, cp, cc, [20]), dim=2)
    assert torch.equal(y, y_off)
    with pytest.raises(fb.FacError):
        fb.VoiceConversionStream(m, 33, torch.zeros(33, 1024, device="cuda:0"))


@pytest.mark.gpu
def test_vc_stream_error_paths(built_lib):
    import facodec_b200 as fb
    from facodec_b200.modules import _ptr, _stream
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    dev = torch.device("cuda:0")
    L, h = m.encoder._engine.L, m.encoder._engine.handle
    cp, cc, tv = _dev_codes(1, 60, 9)
    y_off = fb.VoiceConverter(m).convert([cp, cc], tv)
    part = lambda lo, hi: [cp[:, :, lo:hi], cc[:, :, lo:hi]]
    with fb.VoiceConversionStream(m, 1, tv) as s:
        with pytest.raises(fb.FacError):
            s.finish()                                           # nothing received
        with pytest.raises(fb.FacError):
            s.convert([cp[:, :, :5].cpu(), cc[:, :, :5]])        # CPU tensor
        with pytest.raises(ValueError):
            s.convert(part(0, 0))                                # no frames
        with pytest.raises(ValueError):
            s.convert([cp.repeat(2, 1, 1)[:, :, :5], cc.repeat(2, 1, 1)[:, :, :5]])   # batch mismatch
        bad = cc[:, :, :5].clone()
        bad[0, 0, 2] = 1024
        with pytest.raises(IndexError):
            s.convert([cp[:, :, :5], bad])
        y = torch.empty(300 * 5, device=dev)
        st = _stream(dev)
        assert L.fac_vc_stream_convert(h, s.sid, _ptr(cp), _ptr(cc), 2, 0, _ptr(y), st) == -1    # F = 0
        assert L.fac_vc_stream_convert(h, s.sid, _ptr(cp), _ptr(cc), 0, 5, _ptr(y), st) == -1    # n_c = 1 > 0 rows
        assert L.fac_vc_stream_convert(h, s.sid + 100, _ptr(cp), _ptr(cc), 2, 5, _ptr(y), st) == -1
        # the rejected calls left the stream as it was
        ys = [s.convert(part(0, 30)), s.convert(part(30, 60)), s.finish()]
        with pytest.raises(fb.FacError):
            s.convert(part(0, 5))                                # after finish
        with pytest.raises(fb.FacError):
            s.finish()
    assert torch.equal(torch.cat(ys, dim=2), y_off)
    with pytest.raises(fb.FacError):
        s.convert(part(0, 5))                                    # closed
    with pytest.raises(fb.FacError):
        fb.VoiceConversionStream(m, 1, tv, n_c=3)
    with pytest.raises(fb.FacError):
        fb.VoiceConversionStream(m, 1, tv.cpu())
    with pytest.raises(ValueError):
        fb.VoiceConversionStream(m, 2, tv)

    # out-of-range codes: IndexError on the Python surface, as F.embedding; NaN (never a read past the table) in C
    bad = cc.clone()
    bad[0, 0, 20] = -1
    with pytest.raises(IndexError):
        fb.VoiceConverter(m).convert([cp, bad], tv)
    with pytest.raises(IndexError):
        m.encoder(cp, bad, tv, use_p_code=False, n_c=1)
    with pytest.raises(IndexError):
        with fb.VoiceConversionStream(m, 1, tv) as s:
            s.convert([cp, bad])
    y = torch.zeros(1, 1, 300 * 60, device=dev)
    assert L.fac_voice_convert(h, _ptr(cp), _ptr(bad), 2, _ptr(tv), 1, 60, 0, 1, 1, _ptr(y), _stream(dev)) == 0
    assert not bool(torch.isfinite(y).all())
    bad[0, 0, 20] = 5000
    sid = L.fac_vc_stream_begin(h, 1, _ptr(tv), 0, 1, 1, _stream(dev))
    assert sid >= 0
    try:
        y1, y2 = torch.zeros(300 * 60, device=dev), torch.zeros(300 * 44, device=dev)
        k1 = L.fac_vc_stream_convert(h, sid, _ptr(cp), _ptr(bad), 2, 60, _ptr(y1), _stream(dev))
        k2 = L.fac_vc_stream_finish(h, sid, _ptr(y2), _stream(dev))
        assert (k1, k2) == (16, 44)
        assert not bool(torch.isfinite(torch.cat([y1[:300 * k1], y2])).all())
    finally:
        L.fac_vc_stream_end(h, sid)
    # valid codes still convert as before on the same handle
    assert torch.equal(fb.VoiceConverter(m).convert([cp, cc], tv), y_off)
