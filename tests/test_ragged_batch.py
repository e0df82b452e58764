"""Ragged batches: Codec.encode / forward(lengths=), Codec.decode(frames=) and VoiceConverter.convert(frames=) take
utterances of different lengths in one batch, and each utterance must come out bit-identical to its own B = 1 call on
x[b, :, :lengths[b]] or codes[..., :frames[b]].

What makes that hold: every conv pads each lane about its OWN end (PadMap::lane: reflection, the pad1d short-input zero
extension, the strided convs' right padding, zero padding of the GLU and transposed convs), the STFT reflects each lane
about its own end, the StyleEncoder attends over and pools each lane's own frames in the attention variant its own call
takes, the dequantize / redecoder embedding read no code past a lane's frames, and the outputs past a lane's end are
zeroed (codes: -1).  Host tests pin the per-lane pad map against pad1d on each lane's own sequence and the argument
checks; GPU tests hold the public calls to bit-identity with their B = 1 calls.
"""
import ctypes

import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, load_golden
from oracle import facodec_oracle as O

HOP = 300


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    new = ("fac_codes_decode_lens", "fac_voice_convert_lens", "fac_codec_encode_lens", "fac_codec_forward_lens")
    assert set(new) <= set(_declared("facodec_b200.h"))
    assert "fac_debug_lane_pad_map" in _declared("facodec_b200_debug.h")
    assert set(new) | {"fac_debug_lane_pad_map"} <= set(_lib.EXPORTED)


def _geometries():
    """(pad_left, pad_right, reflect) of every padded conv: the k = 7 convs at dilations 1, 3, 9 (causal in the encoder and
    the codec decoder, centred in the redecoder's decoder), the 2- / 3-tap transposed convs, the redecoder's WaveNet
    (k = 5 centred), the prosody WaveNet (k = 5 causal), the StyleEncoder's GLU convs (k = 5, zeros), the STFT (600 each
    side), and the encoder's stride-s down-sampling convs (k = 2s: s on the left, extra = 0 .. s - 1 on the right)."""
    out = set()
    for k_eff in (7, 19, 55):
        out.add((k_eff - 1, 0, 1))
        out.add(((k_eff - 1) - (k_eff - 1) // 2, (k_eff - 1) // 2, 1))
    out |= {(1, 0, 0), (1, 1, 0), (2, 2, 1), (4, 0, 1), (2, 2, 0), (600, 600, 1)}
    for s in (2, 5, 6):
        out |= {(s, extra, 1) for extra in range(s)}
    return sorted(out)


@pytest.mark.parametrize("pl,pr,reflect", _geometries())
def test_lane_pad_map_is_pad1d_of_each_lane(pl, pr, reflect, built_lib):
    from facodec_b200 import _lib
    L = _lib.load()
    mp = max(pl, pr)
    lens = sorted({1, 2, 3, max(mp - 1, 1), mp, mp + 1, mp + 2, 2 * mp + 5})
    Tin = max(lens) + 7
    B, n = len(lens), pl + Tin + pr
    out = (ctypes.c_int * (B * n))()
    arr = (ctypes.c_int * B)(*lens)
    assert L.fac_debug_lane_pad_map(arr, B, Tin, pl, pr, reflect, out, n) == 0
    got = np.array(out[:]).reshape(B, n)
    for b, Lb in enumerate(lens):
        ramp = torch.arange(1, Lb + 1, dtype=torch.float32).view(1, 1, Lb)     # value i + 1 marks source row i
        ref = O._pad1d_reflect(ramp, pl, pr) if reflect else torch.nn.functional.pad(ramp, (pl, pr))
        own = torch.tensor([0.0 if s < 0 else float(s + 1) for s in got[b, :pl + Lb + pr]])
        assert torch.equal(own, ref.view(-1)), (b, Lb)
        rest = got[b, pl + Lb + pr:]                  # positions only rows past the lane's end read: stay in the lane
        assert ((rest == -1) | ((rest >= 0) & (rest < Lb))).all(), (b, Lb)
    full = (ctypes.c_int * (B * n))()
    assert L.fac_debug_lane_pad_map(None, B, Tin, pl, pr, reflect, full, n) == 0
    ref_full = (ctypes.c_int * n)()
    assert L.fac_debug_pad_map(Tin, pl, pr, reflect, ref_full, n) == 0
    assert np.array_equal(np.array(full[:]).reshape(B, n), np.tile(np.array(ref_full[:]), (B, 1)))
    bad = (ctypes.c_int * B)(*([Tin + 1] * B))
    assert L.fac_debug_lane_pad_map(bad, B, Tin, pl, pr, reflect, out, n) == -1


def test_frame_counts_are_checked_on_host():
    from facodec_b200.modules import _codes_args, _lane_counts
    assert _lane_counts([3, 1, 5], 3, 1, 5, "frames") == [3, 1, 5]
    assert _lane_counts(torch.tensor([2, 5], dtype=torch.int32), 2, 1, 5, "frames") == [2, 5]
    assert _lane_counts((np.int64(4),), 1, 1, 5, "frames") == [4]
    for bad in ([0, 3], [3, 6], [3], [3, 3, 3], [2.0, 3], [2.5, 3], [True, 3], torch.tensor([2.0, 3.0]),
                torch.tensor([[2, 3]]), torch.tensor([True, True]), 3, "ab"):
        with pytest.raises(ValueError):
            _lane_counts(bad, 2, 1, 5, "frames")
    ok = lambda ts: None   # noqa: E731  (device placement is checked on the GPU)
    cp, cc, cr = torch.zeros(2, 1, 5, dtype=torch.int64), torch.ones(2, 2, 5, dtype=torch.int64), torch.full((2, 3, 5), 7)
    tb = torch.zeros(2, 1024)
    cc[0, 1, 3:] = 1024                 # past lane 0's 3 frames: neither read nor checked
    cr[1, 2, 4] = -1                    # past lane 1's 4 frames
    assert _codes_args([cp, cc, cr], tb, ok, [3, 4])[5:] == (2, 5)
    with pytest.raises(IndexError):
        _codes_args([cp, cc, cr], tb, ok, [4, 4])
    with pytest.raises(IndexError):
        _codes_args([cp, cc, cr], tb, ok)
    for bad in ([0, 4], [3, 6], [3], [3.0, 4]):
        with pytest.raises(ValueError):
            _codes_args([cp, cc, cr], tb, ok, bad)


def test_down_conv_right_pad_follows_from_the_lane_length():
    """A stride-s down-sampling conv of a lane pads `extra` = the lane's own round-up on the right.  Its output rows read
    padded positions below L + extra only, and reflection about the lane's own end (pad_right does not enter the map)
    gives exactly those values, so the per-lane map needs no per-lane extra."""
    from facodec_b200 import _lib
    Lb = _lib.load()
    for s in (2, 5, 6):
        for L in range(1, 40):
            F = -(-L // s)                   # conv_out_len: ceil(L / s)
            extra = F * s - L
            n = s + L + extra
            got = (ctypes.c_int * n)()
            assert Lb.fac_debug_pad_map(L, s, extra, 1, got, n) == 0
            Tin = L + 9
            lane = (ctypes.c_int * (s + Tin + s - 1))()
            assert Lb.fac_debug_lane_pad_map((ctypes.c_int * 1)(L), 1, Tin, s, s - 1, 1, lane, s + Tin + s - 1) == 0
            assert list(lane[:n]) == list(got[:]), (s, L)


def test_sample_counts_are_checked_on_host():
    from facodec_b200.modules import _lane_counts
    assert _lane_counts([1025, 9000], 2, 1025, 9000, "lengths") == [1025, 9000]
    for bad in ([1024, 9000], [1025, 9001], [5000], [5000.0, 6000], torch.tensor([5000.0, 6000.0])):
        with pytest.raises(ValueError):
            _lane_counts(bad, 2, 1025, 9000, "lengths")


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _codes(B, T, n_c, n_r, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 1024, (B, rows, T), generator=g).cuda() for rows in (1, n_c, n_r)]


def _fill_tails(codes, frames, value_fn):
    """codes with every frame past its lane's end replaced by value_fn(shape) (a new list; inputs untouched)."""
    out = []
    for c in codes:
        c = c.clone()
        for b, f in enumerate(frames):
            if f < c.shape[2] and c.shape[1]:
                c[b, :, f:] = value_fn(c[b, :, f:].shape).to(c.device)
        out.append(c)
    return out


def _timbre(B, seed):
    return (0.3 * torch.randn(B, 1024, generator=torch.Generator().manual_seed(seed))).cuda()


def _check_lanes(y, frames, one):
    """y [B,1,300 T] of a ragged call: lane b equals one(b) bit for bit on its frames and is 0 past them."""
    for b, f in enumerate(frames):
        y1 = one(b)
        assert y1.shape == (1, 1, HOP * f)
        assert torch.equal(y[b:b + 1, :, :HOP * f], y1), f"lane {b} ({f} frames) differs from its own call"
        assert not bool(y[b, :, HOP * f:].any()), f"lane {b}: samples past its end must be 0"


def _decode_case(codec, frames, n_c, n_r, seed):
    B, T = len(frames), max(frames)
    codes = _codes(B, T, n_c, n_r, seed)
    tv = _timbre(B, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    ys = []
    for fill in (lambda s: torch.randint(0, 1024, s, generator=g), lambda s: torch.full(s, 1023),
                 lambda s: torch.full(s, -1)):
        ys.append(codec.decode(_fill_tails(codes, frames, fill), tv, frames=frames))
    torch.cuda.synchronize()
    assert torch.equal(ys[0], ys[1]) and torch.equal(ys[0], ys[2]), "codes past a lane's end must not matter"
    _check_lanes(ys[0], frames, lambda b: codec.decode([c[b:b + 1, :, :frames[b]] for c in codes], tv[b:b + 1]))


@pytest.mark.gpu
@pytest.mark.parametrize("n_c,n_r", [(1, 0), (2, 3), (1, 3), (2, 0)])
def test_decode_frames_match_b1(n_c, n_r, built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    # full-length lane, the first conv's short-input branch (<= 6 frames), the 768-channel stage's (<= 9), one frame
    _decode_case(codec, [40, 6, 3, 9, 10, 1, 23, 5], n_c, n_r, seed=10 * n_c + n_r)


@pytest.mark.gpu
def test_decode_many_lanes(built_lib):
    """35 lanes: more than the 32 sequences of one LSTM launch and one per-lane dequantize launch."""
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    frames = [1 + (7 * b) % 12 for b in range(35)]
    frames[17] = 14
    _decode_case(codec, frames, 2, 3, seed=77)


@pytest.mark.gpu
def test_decode_equal_frames_change_nothing(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    codes, tv = _codes(3, 17, 2, 3, 5), _timbre(3, 6)
    y0 = codec.decode(codes, tv)
    n0 = codec.launch_count()
    y1 = codec.decode(codes, tv, frames=torch.tensor([17, 17, 17]))
    n1 = codec.launch_count()
    torch.cuda.synchronize()
    assert torch.equal(y0, y1) and n0 == n1


@pytest.mark.gpu
def test_decode_fma_path(built_lib):
    """tensor_cores = 0: every layer on the SIMT kernels, against B = 1 under the same option."""
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    m = model_for(0)
    codec = fb.Codec(m)
    e = codec.engine
    e.set_option("tensor_cores", 0)
    try:
        _decode_case(codec, [12, 4, 9, 1], 1, 3, seed=3)
    finally:
        e.set_option("tensor_cores", 2)


@pytest.mark.gpu
def test_convert_fma_path(built_lib):
    """tensor_cores = 0: the redecoder WaveNet and the 3-tap transposed convs (which read one row past a lane's end) on the
    SIMT kernels, against B = 1 under the same option."""
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    vc = fb.VoiceConverter(redec_model_for(0))
    vc.engine.set_option("tensor_cores", 0)
    try:
        frames = [9, 2, 5, 1]
        B, T = len(frames), max(frames)
        cp, cc, _ = _codes(B, T, 2, 0, seed=12)
        tv = _timbre(B, 13)
        y = vc.convert([cp, cc], tv, use_p_code=True, n_c=2, frames=frames)
        torch.cuda.synchronize()
        _check_lanes(y, frames, lambda b: vc.convert([cp[b:b + 1, :, :frames[b]], cc[b:b + 1, :, :frames[b]]], tv[b:b + 1],
                                                     use_p_code=True, n_c=2))
    finally:
        vc.engine.set_option("tensor_cores", 2)


@pytest.mark.gpu
def test_decode_golden_codes_in_one_ragged_batch(built_lib):
    """The same-weight golden cases' codes packed into one batch: each lane is its own B = 1 decode bit for bit, and
    within the fixtures' waveform bar."""
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    lanes = []
    for name in ("b2_t7200", "b1_t96000", "b1_t7000_ragged"):
        assert GOLDEN_CASES[name]["wseed"] == 0
        g = load_golden(name)
        for b in range(g["codes_p"].shape[0]):
            lanes.append(([torch.from_numpy(g[k][b:b + 1]) for k in ("codes_p", "codes_c", "codes_r")],
                          torch.from_numpy(g["timbre"][b:b + 1]), g["y"][b:b + 1]))
    frames = [l[0][0].shape[2] for l in lanes]
    T = max(frames)
    codes = [torch.cat([torch.nn.functional.pad(l[0][i], (0, T - l[0][i].shape[2]), value=512) for l in lanes]).cuda()
             for i in range(3)]
    tv = torch.cat([l[1] for l in lanes]).cuda()
    y = codec.decode(codes, tv, frames=frames)
    torch.cuda.synchronize()
    _check_lanes(y, frames, lambda b: codec.decode([c[b:b + 1, :, :frames[b]] for c in codes], tv[b:b + 1]))
    for b, l in enumerate(lanes):
        ref = torch.from_numpy(l[2]).double()
        rms = float(((y[b:b + 1, :, :HOP * frames[b]].cpu().double() - ref) ** 2).mean().sqrt())
        assert rms <= 1e-4, (b, rms)


@pytest.mark.gpu
@pytest.mark.parametrize("use_p,n_c", [(False, 1), (True, 1), (False, 2), (True, 2)])
def test_convert_frames_match_b1(use_p, n_c, built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    vc = fb.VoiceConverter(redec_model_for(0))
    frames = [50, 2, 5, 13, 1, 33, 44]
    B, T = len(frames), max(frames)
    cp, cc, _ = _codes(B, T, 2, 0, seed=40 + n_c)
    tv = _timbre(B, 41)
    g = torch.Generator().manual_seed(42)
    ys = [vc.convert(_fill_tails([cp, cc], frames, fill), tv, use_p_code=use_p, n_c=n_c, frames=frames)
          for fill in (lambda s: torch.randint(0, 1024, s, generator=g), lambda s: torch.zeros(s, dtype=torch.int64))]
    torch.cuda.synchronize()
    assert torch.equal(ys[0], ys[1]), "codes past a lane's end must not matter"
    _check_lanes(ys[0], frames, lambda b: vc.convert([cp[b:b + 1, :, :frames[b]], cc[b:b + 1, :, :frames[b]]], tv[b:b + 1],
                                                     use_p_code=use_p, n_c=n_c))


@pytest.mark.gpu
def test_convert_many_lanes_and_equal_frames(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    vc = fb.VoiceConverter(redec_model_for(0))
    frames = [1 + (5 * b) % 11 for b in range(35)]
    B, T = len(frames), max(frames)
    cp, cc, _ = _codes(B, T, 1, 0, seed=9)
    tv = _timbre(B, 10)
    y = vc.convert([cp, cc], tv, frames=frames)
    torch.cuda.synchronize()
    _check_lanes(y, frames, lambda b: vc.convert([cp[b:b + 1, :, :frames[b]], cc[b:b + 1, :, :frames[b]]], tv[b:b + 1]))
    y0 = vc.convert([cp, cc], tv)
    n0 = vc.engine.L.fac_last_launch_count(vc.engine.handle)
    y1 = vc.convert([cp, cc], tv, frames=[T] * B)
    n1 = vc.engine.L.fac_last_launch_count(vc.engine.handle)
    torch.cuda.synchronize()
    assert torch.equal(y0, y1) and n0 == n1


@pytest.mark.gpu
def test_c_abi_rejects_bad_frame_counts(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    codes, tv = _codes(2, 8, 1, 0, 1), _timbre(2, 2)
    codec.decode(codes, tv)                   # weights synced
    e = codec.engine
    y = torch.empty(2, 1, 8 * HOP, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    for bad in ([0, 8], [8, 9], [-3, 2]):
        rc = e.L.fac_codes_decode_lens(e.handle, p(codes[0]), p(codes[1]), 1, None, 0, p(tv), 2, 8, (ctypes.c_int * 2)(*bad),
                                       p(y), None)
        assert rc == -1 and b"frames" in e.L.fac_last_error(e.handle), bad
    with pytest.raises(ValueError):
        codec.decode(codes, tv, frames=[8])


# ---------------------------------------------------------------------------------------------------------------------
# GPU: encode / forward
# ---------------------------------------------------------------------------------------------------------------------
def _ragged_waves(lengths, T, seed, pad_seed, amp=50.0):
    """[B,1,T]: lane b's first lengths[b] samples from synth_waves (its own seed), the rest large seeded finite noise."""
    from facodec_b200 import synth
    x = torch.empty(len(lengths), 1, T)
    g = torch.Generator().manual_seed(pad_seed)
    for b, L in enumerate(lengths):
        x[b, :, :L] = synth.synth_waves(1, L, seed=seed + b)[0]
        x[b, :, L:] = amp * torch.randn(1, T - L, generator=g)
    return x.cuda()


def _check_encode_lanes(codec, x, lengths, codes, timbre, y=None):
    """codes / timbre (/ y) of a ragged call: lane b bit-equal to its own B = 1 call on its own samples; past its end,
    codes are -1 and y is 0."""
    import facodec_b200 as fb
    Tq = codes[0].shape[2]
    for b, L in enumerate(lengths):
        xb = x[b:b + 1, :, :L].contiguous()
        if y is None:
            c1, t1 = codec.encode(xb, n_c=codes[1].shape[1])
        else:
            y1, c1, t1 = codec.forward(xb, n_c=codes[1].shape[1])
        F = c1[0].shape[2]
        assert F == min(L // HOP, fb.Codec(codec.model).engine.L.fac_encode_frames(L))
        for got, ref in zip(codes, c1):
            assert torch.equal(got[b:b + 1, :, :F], ref), f"lane {b} ({L} samples): codes differ"
            assert bool((got[b, :, F:Tq] == -1).all()), f"lane {b}: codes past its end must be -1"
        assert torch.equal(timbre[b:b + 1], t1), f"lane {b} ({L} samples): timbre differs"
        if y is not None:
            assert torch.equal(y[b:b + 1, :, :HOP * F], y1), f"lane {b} ({L} samples): y differs"
            assert not bool(y[b, :, HOP * F:].any()), f"lane {b}: y past its end must be 0"


LENGTHS = [9000, 6000, 7000, 1500, 1025, 2600]   # full, a multiple of 300, a non-multiple, short, the shortest, the
                                                 # 512-channel stage's short-input branch (T / 50 <= 54 rows)


@pytest.mark.gpu
@pytest.mark.parametrize("call", ["encode", "forward"])
def test_encode_forward_lengths_match_b1(call, built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    T = max(LENGTHS)
    outs = []
    for pad_seed, order in ((1, list(range(len(LENGTHS)))), (2, [3, 0, 5, 1, 4, 2])):
        lengths = [LENGTHS[i] for i in order]
        x = _ragged_waves(LENGTHS, T, seed=500, pad_seed=pad_seed)[order]
        if call == "encode":
            codes, timbre = codec.encode(x, n_c=2, lengths=lengths)
            y = None
        else:
            y, codes, timbre = codec.forward(x, n_c=2, lengths=torch.tensor(lengths))
        torch.cuda.synchronize()
        _check_encode_lanes(codec, x, lengths, codes, timbre, y)
        inv = [order.index(i) for i in range(len(order))]
        outs.append([t[inv] for t in codes] + [timbre[inv]] + ([] if y is None else [y[inv]]))
    assert all(torch.equal(a, b) for a, b in zip(*outs)), "padding or lane order changed a lane's bits"


@pytest.mark.gpu
def test_encode_equal_lengths_change_nothing(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    x = _ragged_waves([4800] * 3, 4800, seed=7, pad_seed=0)
    y0, c0, t0 = codec.forward(x)
    n0 = codec.launch_count()
    y1, c1, t1 = codec.forward(x, lengths=[4800] * 3)
    n1 = codec.launch_count()
    torch.cuda.synchronize()
    assert torch.equal(y0, y1) and torch.equal(t0, t1) and all(torch.equal(a, b) for a, b in zip(c0, c1)) and n0 == n1


@pytest.mark.gpu
def test_encode_many_lanes_and_fma_path(built_lib):
    """35 lanes (past 32 sequences per LSTM launch); then a small case under tensor_cores = 0 (SPEC mel path, SIMT convs)."""
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    lengths = [1025 + 97 * b for b in range(35)]
    x = _ragged_waves(lengths, max(lengths), seed=900, pad_seed=3)
    codes, timbre = codec.encode(x, n_c=1, lengths=lengths)
    torch.cuda.synchronize()
    _check_encode_lanes(codec, x, lengths, codes, timbre)
    codec.engine.set_option("tensor_cores", 0)
    try:
        lengths = [3000, 1025, 2000]
        x = _ragged_waves(lengths, 3000, seed=950, pad_seed=4)
        y, codes, timbre = codec.forward(x, n_c=2, lengths=lengths)
        torch.cuda.synchronize()
        _check_encode_lanes(codec, x, lengths, codes, timbre, y)
    finally:
        codec.engine.set_option("tensor_cores", 2)


@pytest.mark.gpu
def test_encode_long_lane_past_the_attention_switch(built_lib):
    """One lane of 2800 mel frames (its own call attends with recomputed scores) beside short lanes (stored scores)."""
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    lengths = [840000, 30000, 3000]
    x = _ragged_waves(lengths, 840000, seed=70, pad_seed=5, amp=5.0)
    codes, timbre = codec.encode(x, n_c=2, lengths=lengths)
    torch.cuda.synchronize()
    _check_encode_lanes(codec, x, lengths, codes, timbre)


@pytest.mark.gpu
def test_encode_golden_inputs_in_one_ragged_batch(built_lib):
    """The same-weight golden cases' inputs packed into one batch: codes equal the fixtures bit for bit, timbre and y
    within their bars."""
    import facodec_b200 as fb
    from conftest import case_inputs
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    lanes = []
    for name in ("b2_t7200", "b1_t96000", "b1_t7000_ragged"):
        c = GOLDEN_CASES[name]
        g = load_golden(name)
        x, _ = case_inputs(c)
        for b in range(c["B"]):
            lanes.append((x[b:b + 1], {k: g[k][b:b + 1] for k in ("codes_p", "codes_c", "codes_r", "timbre", "y")}))
    lengths = [l[0].shape[2] for l in lanes]
    T = max(lengths)
    x = torch.cat([torch.nn.functional.pad(l[0], (0, T - l[0].shape[2]), value=0.5) for l in lanes]).cuda()
    y, codes, timbre = codec.forward(x, n_c=2, lengths=lengths)
    torch.cuda.synchronize()
    for b, (_, g) in enumerate(lanes):
        F = g["codes_p"].shape[2]
        for k, t in zip(("codes_p", "codes_c", "codes_r"), codes):
            assert np.array_equal(t[b:b + 1, :, :F].cpu().numpy(), g[k]), (b, k)
        assert np.abs(timbre[b:b + 1].cpu().numpy() - g["timbre"]).max() <= 1e-5 * max(1.0, np.abs(g["timbre"]).max())
        rms = float(((y[b:b + 1, :, :HOP * F].cpu().double() - torch.from_numpy(g["y"]).double()) ** 2).mean().sqrt())
        assert rms <= 1e-4, (b, rms)


@pytest.mark.gpu
def test_c_abi_rejects_bad_sample_counts(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(0))
    x = _ragged_waves([3000, 3000], 3000, seed=1, pad_seed=1)
    codec.encode(x)                           # weights synced
    e = codec.engine
    cs = [torch.empty(2, r, 10, dtype=torch.int64, device="cuda") for r in (1, 2, 3)]
    p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    for bad in ([1024, 3000], [3000, 3001]):
        rc = e.L.fac_codec_encode_lens(e.handle, p(x), 2, 3000, (ctypes.c_int * 2)(*bad), 2, *map(p, cs), None, None)
        assert rc == -1 and b"lengths" in e.L.fac_last_error(e.handle), bad
    with pytest.raises(ValueError):
        codec.forward(x, lengths=[3000, 1024])
