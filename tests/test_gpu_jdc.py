"""JDCNet (eval mode) and train.py's F0 / energy targets on the GPU against the fp64 restatement in oracle/jdc_oracle.py.

Bars follow the other fp64 tests: a multiple of the fp32 CPU error of the same computation on the same inputs (the 3x3
convs, the input GEMMs and the recurrence run in the fp32-faithful promoted classes), with a floor for outputs the fp32
run happens to reproduce almost exactly.
"""
import ctypes

import pytest
import torch

import facodec_b200 as fb
from facodec_b200 import synth
from oracle import jdc_oracle as O

pytestmark = pytest.mark.gpu

BAR = 16.0


def _mel(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    # normalized log-mel ((log mel + 4) / 4): mostly in [-2, 1]
    return (torch.randn(B, 1, 80, T, generator=g) * 0.6 - 0.5).float()


def _check(name, got, ref64, ref32, floor=1e-6):
    got = got.detach().cpu().double()
    err = (got - ref64).abs().max().item()
    e32 = (ref32.double() - ref64).abs().max().item()
    bar = BAR * e32 + floor * max(1.0, ref64.abs().max().item())
    assert err <= bar, f"{name}: max err {err:.3e} > bar {bar:.3e} (fp32 err {e32:.3e})"
    return err, bar


@pytest.fixture(scope="module")
def sd():
    return synth.synth_jdc(0)


@pytest.fixture(scope="module")
def net(sd):
    m = fb.JDCNet()
    m.load_state_dict(sd)
    return m.eval()


def test_whole_forward_against_fp64(net, sd):
    x = _mel(2, 160, 1)
    f0, gan, pool = net(x.cuda())
    torch.cuda.synchronize()
    r64 = O.jdc_forward(sd, x)
    r32 = O.jdc_forward(sd, x, dtype=torch.float32)
    assert f0.shape == (2, 160) and gan.shape == (2, 256, 10, 160) and pool.shape == (2, 256, 160, 2)
    err, bar = _check("F0", f0, r64[0], r32[0])
    _check("GAN_feature", gan, r64[1], r32[1])
    _check("poolblock_out", pool, r64[2], r32[2])
    # the voiced decision agrees wherever the fp64 F0 is not within the bar of 5.0
    ref = r64[0]
    far = (ref - 5.0).abs() > bar
    assert far.any() and (ref > 5.0).any() and (ref <= 5.0).any()
    assert torch.equal((f0.cpu().double() > 5.0)[far], (ref > 5.0)[far])


def _taps(net, names, x, lengths=None):
    e = net._engine
    net._sync(x.device)
    B, T = x.shape[0], x.shape[-1]
    size = {"jdc.conv_in": 82 * 64, "jdc.conv_block": 82 * 64, "jdc.res1.pre": 42 * 64, "jdc.res1.conv1": 42 * 128,
            "jdc.res1": 42 * 128, "jdc.res2.pre": 22 * 128, "jdc.res2.conv1": 22 * 192, "jdc.res2": 22 * 192,
            "jdc.res3.pre": 12 * 192, "jdc.res3.conv1": 12 * 256, "jdc.res3": 12 * 256, "jdc.lstm_in": 512,
            "jdc.lstm.fwd": 256, "jdc.lstm.rev": 256}
    bufs = {n: torch.full((B * T * size[n],), float("nan"), device=x.device) for n in names}
    for n, b in bufs.items():
        assert e.L.fac_debug_tap(e.handle, n.encode(), ctypes.c_void_p(b.data_ptr()), b.numel()) == 0
    try:
        net(x, lengths)
        torch.cuda.synchronize()
    finally:
        for n in names:
            e.L.fac_debug_tap(e.handle, n.encode(), None, 0)
    return {n: b.cpu() for n, b in bufs.items()}


def _nchw(buf, B, T, F, C):
    """[B][T][F + 2][C] map with pad columns -> NCHW [B, C, T, F] as the reference holds it (pad columns must be 0)."""
    m = buf.reshape(B, T, F + 2, C)
    assert torch.all(m[:, :, 0] == 0) and torch.all(m[:, :, F + 1] == 0), "pad columns are not zero"
    return m[:, :, 1:F + 1].permute(0, 3, 1, 2).double()


def test_each_block_teacher_forced(net, sd):
    """Each conv / ResBlock / pool / LSTM direction from the engine's own input tap, against fp64 and its fp32 twin."""
    import torch.nn.functional as Fn
    B, T = 1, 96
    x = _mel(B, T, 2)
    names = ["jdc.conv_in", "jdc.conv_block", "jdc.res1.pre", "jdc.res1.conv1", "jdc.res1", "jdc.res2.pre", "jdc.res2.conv1",
             "jdc.res2", "jdc.res3.pre", "jdc.res3.conv1", "jdc.res3", "jdc.lstm_in", "jdc.lstm.fwd", "jdc.lstm.rev"]
    tp = _taps(net, names, x.cuda())
    chans = {"jdc.conv_in": (80, 64), "jdc.conv_block": (80, 64), "jdc.res1.pre": (40, 64), "jdc.res1.conv1": (40, 128),
             "jdc.res1": (40, 128), "jdc.res2.pre": (20, 128), "jdc.res2.conv1": (20, 192), "jdc.res2": (20, 192),
             "jdc.res3.pre": (10, 192), "jdc.res3.conv1": (10, 256), "jdc.res3": (10, 256)}
    m = {n: _nchw(tp[n], B, T, *chans[n]) for n in chans}
    ref = {}
    for dt in (torch.float64, torch.float32):
        xi = x.to(dt).transpose(-1, -2)
        r = {"jdc.conv_in": O._lrelu(O._bn(sd, "conv_block.1", O._conv(sd, "conv_block.0.weight", xi, 1)))}
        r["jdc.conv_block"] = O._conv(sd, "conv_block.3.weight", m["jdc.conv_in"].to(dt), 1)
        prev = "jdc.conv_block"
        for i, (name, _, _) in enumerate(O._BLOCKS):
            k = "jdc.res%d" % (i + 1)
            r[k + ".pre"] = Fn.max_pool2d(O._lrelu(O._bn(sd, name + ".pre_conv.0", m[prev].to(dt))), (1, 2))
            r[k + ".conv1"] = O._lrelu(O._bn(sd, name + ".conv.1", O._conv(sd, name + ".conv.0.weight", m[k + ".pre"].to(dt), 1)))
            r[k] = (O._conv(sd, name + ".conv.3.weight", m[k + ".conv1"].to(dt), 1)
                    + O._conv(sd, name + ".conv1by1.weight", m[k + ".pre"].to(dt), 0))
            prev = k
        p = Fn.max_pool2d(O._lrelu(O._bn(sd, "pool_block.0", m["jdc.res3"].to(dt))), (1, 4))
        r["jdc.lstm_in"] = p.permute(0, 2, 1, 3).reshape(T, 512)
        seq = tp["jdc.lstm_in"].reshape(T, 512).to(dt)
        for sfx, rev, key in (("_l0", False, "jdc.lstm.fwd"), ("_l0_reverse", True, "jdc.lstm.rev")):
            w = [sd["bilstm_classifier." + n + sfx].to(dt) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
            r[key] = O.lstm_dir(*w, seq, reverse=rev)
        ref[dt] = r
    got = dict(m)
    for n in ("jdc.lstm_in", "jdc.lstm.fwd", "jdc.lstm.rev"):
        got[n] = tp[n].reshape(T, -1)
    for n in names:
        _check(n, got[n], ref[torch.float64][n].double(), ref[torch.float32][n])


def test_ragged_lanes_equal_their_own_calls(net, sd):
    T = 203
    lens = [203, 1, 77, 130]             # 77 and 130 frames: no multiple of any tile or of F + 2
    x = _mel(4, T, 3).cuda()
    f0, gan, pool = net(x, lens)
    for b, L in enumerate(lens):
        f1, g1, p1 = net(x[b:b + 1, :, :, :L].contiguous())
        assert torch.equal(f0[b, :L], f1[0]), f"lane {b}: F0 differs from its B = 1 call"
        assert torch.equal(gan[b, :, :, :L], g1[0]) and torch.equal(pool[b, :, :L], p1[0])
        assert torch.all(f0[b, L:] == 0) and torch.all(gan[b, :, :, L:] == 0) and torch.all(pool[b, :, L:] == 0)
    r64 = O.jdc_forward(sd, x.cpu(), lens)
    r32 = O.jdc_forward(sd, x.cpu(), lens, dtype=torch.float32)
    _check("ragged F0", f0, r64[0], r32[0])


def test_batch_tail_and_lengths(net, sd):
    """B = 33 (a second LSTM group of one lane), equal to its lanes' B = 1 calls; T from 1 to 3000 frames against fp64;
    a ragged pair of about 3000 frames, each lane equal to its own B = 1 call."""
    x = _mel(33, 40, 4).cuda()
    f0, _, _ = net(x)
    for b in (0, 31, 32):
        assert torch.equal(f0[b], net(x[b:b + 1])[0][0])
    for T in (1, 2, 3000):
        xt = _mel(1, T, 5 + T)
        f, g, p = net(xt.cuda())
        torch.cuda.synchronize()
        assert f.shape == (1, T)
        r64 = O.jdc_forward(sd, xt)
        r32 = O.jdc_forward(sd, xt, dtype=torch.float32)
        _check("F0 T=%d" % T, f, r64[0], r32[0])
        _check("GAN_feature T=%d" % T, g, r64[1], r32[1])
        _check("poolblock_out T=%d" % T, p, r64[2], r32[2])
    lens = [3000, 2937]
    x2 = _mel(2, 3000, 9).cuda()
    f2, g2, p2 = net(x2, lens)
    for b, L in enumerate(lens):
        f1, g1, p1 = net(x2[b:b + 1, :, :, :L].contiguous())
        assert torch.equal(f2[b, :L], f1[0]) and torch.equal(g2[b, :, :, :L], g1[0]) and torch.equal(p2[b, :, :L], p1[0])


def test_pinned_reference_inputs():
    """The mels and F0 rows of pin_jdc.npz (the unmodified reference's outputs, oracle/make_jdc_golden.py)."""
    import os
    import numpy as np
    pin = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pin_jdc.npz"))
    sd = synth.synth_jdc(int(pin["seed"]))
    net = fb.JDCNet()
    net.load_state_dict(sd)
    net.eval()
    for i in range(len(pin["cases"])):
        x = torch.from_numpy(pin[f"mel_{i}"])
        f0, gan, pool = net(x.cuda())
        r64 = O.jdc_forward(sd, x)
        r32 = O.jdc_forward(sd, x, dtype=torch.float32)
        ref = torch.from_numpy(pin[f"f0_{i}"]).double()
        # the reference's fp32 run is one more fp32 computation: within its own distance of fp64 plus the bar
        bar = BAR * (r32[0].double() - r64[0]).abs().max().item() + (ref - r64[0]).abs().max().item() + 1e-6 * ref.abs().max().item()
        assert (f0.cpu().double() - ref).abs().max().item() <= bar
        _check("pin GAN_feature %d" % i, gan, r64[1], r32[1])
        _check("pin poolblock_out %d" % i, pool, r64[2], r32[2])
    tg, glob = fb.f0_targets(torch.from_numpy(pin["targets_f0"]).cuda())
    rtg, rglob = torch.from_numpy(pin["targets"]).double(), torch.from_numpy(pin["targets_glob"]).double()
    assert torch.equal(tg.cpu() == -10.0, rtg == -10.0) and (tg.cpu().double() - rtg).abs().max().item() <= 1e-4
    fin = torch.isfinite(rglob)
    assert torch.equal(fin, torch.isfinite(glob.cpu())) and (glob.cpu().double()[fin] - rglob[fin]).abs().max().item() <= 1e-5


def test_errors(net):
    x = _mel(1, 16, 6)
    with pytest.raises(fb.FacError):
        net(x)                                # CPU tensor
    with pytest.raises(fb.FacError):
        net(torch.zeros(1, 1, 64, 16, device="cuda"))
    with pytest.raises(ValueError):
        net(x.cuda(), [17])
    m = fb.JDCNet()
    with pytest.raises(NotImplementedError):
        m.train()(x.cuda())
    with pytest.raises(fb.FacError):
        fb.f0_targets(torch.ones(2, 5))
    with pytest.raises(fb.FacError):
        fb.log_norm(torch.zeros(1, 1, 80, 4))


def test_f0_targets_against_fp64():
    g = torch.Generator().manual_seed(7)
    T = 300
    f0 = torch.rand(6, T, generator=g) * 400.0
    f0[f0 < 80.0] = 0.0                      # unvoiced frames
    f0[1] = 0.0                              # no voiced frame
    f0[2] = 0.0
    f0[2, 17] = 220.0                        # exactly one voiced frame: std NaN -> -10, mean kept
    f0[3, 5] = float("inf")                  # an inf F0: the mean turns inf / NaN -> every voiced frame -10
    f0[4, :] = 8.0                           # all frames equal (log2 exact): std 0, 0 / 0 -> -10
    out, glob = fb.f0_targets(f0.cuda())
    ref, rglob = O.f0_targets(f0)
    out, glob = out.cpu().double(), glob.cpu().double()
    assert torch.equal(out == -10.0, ref == -10.0)
    assert (out - ref).abs().max().item() <= 1e-4
    fin = torch.isfinite(rglob)
    assert torch.equal(fin, torch.isfinite(glob))
    assert (glob[fin] - rglob[fin]).abs().max().item() <= 1e-5
    assert glob[1] == 0.0 and out[1].eq(-10.0).all()
    assert abs(glob[2].item() - torch.tensor(220.0).log2().item()) < 1e-5 and out[2].eq(-10.0).all()
    # ragged lengths: lane b over its first lengths[b] frames, -10 after; equal to the trimmed B = 1 call
    lens = [T, 0, 18, 150, 1, 299]
    out_l, glob_l = fb.f0_targets(f0.cuda(), lens)
    ref_l, rglob_l = O.f0_targets(f0, lens)
    assert torch.equal(out_l.cpu() == -10.0, ref_l == -10.0)
    for b, L in enumerate(lens):
        if L:
            o1, g1 = fb.f0_targets(f0[b:b + 1, :L].cuda())
            assert torch.equal(o1[0], out_l[b, :L]) and torch.equal(g1[0], glob_l[b])
    same, glob_none = fb.f0_targets(f0.cuda(), norm_f0=False)
    assert glob_none == [] and torch.equal(same.cpu(), f0)


def test_log_norm_against_fp64():
    mel = _mel(3, 250, 8)
    out = fb.log_norm(mel.cuda())                # [B, 1, 80, T], dim 2 -> [B, 1, T]
    assert out.shape == (3, 1, 250)
    ref = O.log_norm(mel[:, 0])
    r32 = torch.log(torch.exp(mel[:, 0] * 4 - 4).norm(dim=1))
    _check("log_norm", out[:, 0], ref, r32)
    out3 = fb.log_norm(mel[:, 0].cuda(), dim=1)
    assert torch.equal(out3, out[:, 0])
    big = torch.full((1, 80, 3), 30.0)           # exp(116) squared overflows fp32: inf, as the reference's fp32 norm
    assert torch.isinf(fb.log_norm(big.cuda(), dim=1)).all()
