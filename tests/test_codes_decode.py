"""Decoding from codes (FAquantizer.from_codes, Codec.decode, CodecStream.decode_codes) and compress-only encoding
(Codec.encode).

The reference has no single call for it; the semantics are ResidualVectorQuantize.from_codes (dac/nn/quantize.py:200-220)
of the prosody, content and residual quantizers, then the AdaLN of FAquantizer.forward_v2 (modules/quantize.py:437-449),
pinned by tests/golden/pin_from_codes.npz (python -m oracle.from_codes).  CPU tests check the oracle against that
pin and the fixtures; GPU tests check dequantize_kernel against an fp64 restatement with elementwise rounding bounds and
the public calls against the fixtures, the forward, the oracle and the stream.
"""
import ctypes

import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, load_golden, state_dicts
from oracle import facodec_oracle as O
from oracle import from_codes as FC
from test_oracle import _close, _pin

PIN_CASES = ("codec", "c1r3", "c2r1", "c2r0")
RMS_TOL = 1e-4          # north_star: reconstructed waveform within 1e-4 RMS


def _pin_case(pin, name):
    return {k.split("/", 1)[1]: torch.from_numpy(v) for k, v in pin.items() if k.startswith(name + "/")}


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_pin_case_table():
    pin = _pin("from_codes")
    for n_c, n_r in FC.RANDOM_ROWS:
        c = _pin_case(pin, f"c{n_c}r{n_r}")
        codes, timbre = FC.random_case(n_c, n_r)
        for k, t in zip(("codes_p", "codes_c", "codes_r"), codes):
            assert torch.equal(c[k], t), k
            if t.shape[1]:
                assert int(t.min()) == 0 and int(t.max()) == 1023, k
        assert torch.equal(c["timbre"], timbre)
    g = _pin("codec")
    c = _pin_case(pin, "codec")
    for k in ("codes_p", "codes_c", "codes_r", "timbre"):
        assert np.array_equal(c[k].numpy(), g[k]), k


@pytest.mark.parametrize("name", PIN_CASES)
def test_oracle_from_codes_matches_imported_reference(name):
    c = _pin_case(_pin("from_codes"), name)
    sds = state_dicts(1)
    outs, parts = FC.quantizer_from_codes(sds["quantizer"], c["codes_p"], c["codes_c"], c["codes_r"], c["timbre"])
    for k, t in (("outs", outs), ("z_p", parts[0]), ("z_c", parts[1]), ("z_r", parts[2])):
        _close(t, c[k], k)
    with torch.no_grad():
        y = O.decoder_forward(sds["decoder"], outs)
    _close(y, c["y"], "y")


@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_from_codes_close_to_forward(name):
    """from_codes applies out_proj to the raw codebook row, the forward to the straight-through value z_e + (z_q - z_e):
    the two differ in the last bits only."""
    g = load_golden(name)
    sd = state_dicts(GOLDEN_CASES[name]["wseed"])["quantizer"]
    cp, cc, cr, tb = (torch.from_numpy(g[k]) for k in ("codes_p", "codes_c", "codes_r", "timbre"))
    outs, _ = FC.quantizer_from_codes(sd, cp, cc, cr, tb)
    err = float((outs - torch.from_numpy(g["outs"])).abs().max())
    print(f"{name}: from-codes outs vs forward outs max abs {err:.3g}")
    assert err <= 2e-6


def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    new = ("fac_codec_encode", "fac_dequantize", "fac_codes_decode", "fac_stream_decode_codes")
    assert set(new) <= set(_declared("facodec_b200.h"))
    assert set(new) <= set(_lib.EXPORTED)


def test_code_argument_checks_on_host():
    from facodec_b200.modules import _codes_args
    ok = lambda ts: None   # noqa: E731  (device placement is checked on the GPU)
    cp, cc, cr = torch.zeros(2, 1, 5, dtype=torch.int64), torch.ones(2, 2, 5, dtype=torch.int64), torch.full((2, 3, 5), 1023)
    tb = torch.zeros(2, 1024)
    out = _codes_args([cp, cc, cr], tb, ok)
    assert out[3] == 3 and out[5:] == (2, 5)
    assert _codes_args([cp, cc, None], tb, ok)[2:4] == (None, 0)
    assert _codes_args([cp, cc, cr[:, :0]], tb, ok)[2:4] == (None, 0)
    for bad in ([cp, cc], [cp.repeat(1, 2, 1), cc, cr], [cp, cc.repeat(1, 2, 1), cr], [cp, cc, torch.cat([cr, cr[:, :1]], 1)],
                [cp, cc[:1], cr], [cp, cc, cr[:, :, :4]], [cp.float(), cc, cr], [cp[:, :, :0], cc[:, :, :0], None]):
        with pytest.raises(ValueError):
            _codes_args(bad, tb, ok)
    with pytest.raises(ValueError):
        _codes_args([cp, cc, cr], torch.zeros(2, 512), ok)
    for v in (-1, 1024):
        c2 = cc.clone()
        c2[1, 1, 4] = v
        with pytest.raises(IndexError):
            _codes_args([cp, c2, cr], tb, ok)


def test_dac_file_unpack(tmp_path):
    from facodec_b200 import codefile
    g = torch.Generator().manual_seed(3)
    for n_c in (1, 2):
        codes = [torch.randint(0, 1024, (2, n, 11), generator=g) for n in (1, n_c, 3)]
        f = codefile.DACFile.load(codefile.from_forward(codes, original_length=3300).save(tmp_path / f"c{n_c}"))
        back = f.unpack()
        assert [tuple(t.shape) for t in back] == [tuple(t.shape) for t in codes]
        for a, b in zip(back, codes):
            assert a.dtype == torch.int64 and torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _rms(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float(((a - b) ** 2).mean().sqrt())


def _model(seed):
    from test_gpu_parity import model_for
    return model_for(seed)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _random_codes(B, T, n_c, n_r, seed):
    """Random codes with 0 and 1023 in every tensor that has rows (device int64)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for rows in (1, n_c, n_r):
        c = torch.randint(0, 1024, (B, rows, T), generator=g)
        if rows:
            c.view(-1)[0], c.view(-1)[-1] = 0, 1023
        out.append(c.cuda())
    return out


def _dequantize_raw(m, codes, timbre, parts, gb_tap=None):
    """fac_dequantize through the C-ABI: (outs, zp, zc, zr) [B,1024,T] (the parts None when not requested)."""
    cp, cc, cr = codes
    m.quantizer._prep(cp, timbre)
    e = m.quantizer._engine
    B, _, T = cp.shape
    n_r = 0 if cr is None else cr.shape[1]
    outs = torch.full((B, 1024, T), float("nan"), device="cuda")
    zs = [torch.full_like(outs, float("nan")) if parts else None for _ in range(3)]
    if gb_tap is not None:
        assert e.L.fac_debug_tap(e.handle, b"gamma_beta", _p(gb_tap), gb_tap.numel()) == 0
    rc = e.L.fac_dequantize(e.handle, _p(cp), _p(cc), cc.shape[1], _p(cr), n_r, _p(timbre), B, T, _p(outs), *map(_p, zs), None)
    if gb_tap is not None:
        e.L.fac_debug_tap(e.handle, b"gamma_beta", None, 0)
    assert rc == 0, e.L.fac_last_error(e.handle)
    torch.cuda.synchronize()
    return outs, zs


def _fp64_reference(sd, codes, timbre, gb):
    """fp64 z_p, z_c, z_r (the oracle at float64), outs = LayerNorm(s) * gamma + beta with the kernel's own gamma | beta
    (gb [B][2048], read back through the gamma_beta tap), and elementwise bounds on the fp32 kernel's error.

    u = 2^-24, gamma_n = n u / (1 - n u).  Per code, the kernel forms b + sum_k w_k e_k in 8 chained FMAs from the bias:
    error <= gamma_8 (|b| + sum_k |w_k e_k|); the host folds weight-norm in fp32 (g / sqrt, times v: <= 4u |w| per weight
    against the fp64 fold), + 4u sum_k |w_k e_k|.  The RVQ sums and (z_p + z_c) + z_r add at most 5 roundings, each
    <= u times a partial sum bounded by sum |terms|.  The LayerNorm bound is that of test_gpu_quantizer_kernels."""
    from test_gpu_quantizer_kernels import U, gamma
    cp, cc, cr = (None if t is None else t.cpu() for t in codes)
    outs_o, (zp, zc, zr) = FC.quantizer_from_codes(sd, cp, cc, cr, timbre.cpu(), dtype=torch.float64)
    err = {}
    absum = torch.zeros_like(zp)
    for name, prefix, c in (("zp", "prosody_quantizer", cp), ("zc", "content_quantizer", cc), ("zr", "residual_quantizer", cr)):
        e_part = torch.zeros_like(zp)
        a_part = torch.zeros_like(zp)
        for i in range(0 if c is None else c.shape[1]):
            pre = f"{prefix}.quantizers.{i}"
            w = torch._weight_norm(sd[pre + ".out_proj.weight_v"].double(), sd[pre + ".out_proj.weight_g"].double(), 0)[:, :, 0]
            cbrow = sd[pre + ".codebook.weight"].double()[c[:, i, :]]                      # [B][T][8]
            wa = cbrow.abs() @ w.abs().t()                                                 # [B][T][1024]
            ba = sd[pre + ".out_proj.bias"].double().abs()
            e_part += (gamma(8) * (ba + wa) + 4 * U * wa).transpose(1, 2)
            a_part += (ba + wa).transpose(1, 2)
        err[name] = e_part + 2 * U * a_part
        absum += a_part
    s = zp + zc + zr
    eps_s = err["zp"] + err["zc"] + err["zr"] + 5 * U * absum
    mu = s.mean(1, keepdim=True)
    var = (s - mu).pow(2).mean(1, keepdim=True)
    rstd = (var + 1e-5).rsqrt()
    xn = (s - mu) * rstd
    g, b = gb[:, :1024, None].double(), gb[:, 1024:, None].double()
    outs = xn * g + b
    dmu = eps_s.mean(1, keepdim=True) + gamma(37) * s.abs().mean(1, keepdim=True)
    dvar = 2 * ((eps_s + dmu) * (s - mu).abs()).mean(1, keepdim=True) + gamma(38) * var
    rrel = dvar / (2 * (var + 1e-5)) + 2 * U
    dxn = rstd * (eps_s + dmu) + xn.abs() * (rrel + 2 * U)
    douts = g.abs() * dxn + 2 * U * ((g * xn).abs() + b.abs())
    return dict(outs=outs, zp=zp, zc=zc, zr=zr), dict(outs=douts, **err), outs_o


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 17, 320])
@pytest.mark.parametrize("n_c,n_r", [(c, r) for c in (1, 2) for r in (0, 1, 2, 3)])
def test_dequantize_kernel_vs_fp64(n_c, n_r, T, built_lib):
    from test_gpu_quantizer_kernels import U, gamma
    m = _model(0)
    sd = state_dicts(0)["quantizer"]
    B = 3
    codes = _random_codes(B, T, n_c, n_r, seed=100 * n_c + 10 * n_r + T)
    if n_r == 0 and T == 17:
        codes[2] = None                          # no residual tensor at all: same as zero rows
    timbre = (0.3 * torch.randn(B, 1024, generator=torch.Generator().manual_seed(T))).cuda()
    gb = torch.full((B, 2048), float("nan"), device="cuda")
    outs, parts = _dequantize_raw(m, codes, timbre, True, gb_tap=gb)
    outs2, _ = _dequantize_raw(m, codes, timbre, False)
    outs3, parts3 = _dequantize_raw(m, codes, timbre, True)
    assert torch.equal(outs, outs2), "outs must not depend on whether the parts are requested"
    assert torch.equal(outs, outs3) and all(torch.equal(a, b) for a, b in zip(parts, parts3)), "two calls differ"
    gb = gb.cpu().double()
    # gamma | beta: the quantizer-side promoted tensor-core class (22-bit operands, fp32 accumulation over 1024 terms)
    wl, bl = sd["timbre_linear.weight"].double(), sd["timbre_linear.bias"].double()
    tt = timbre.cpu().double()
    gb_ref = tt @ wl.t() + bl
    gb_bound = (2.0 ** -20 + gamma(1025)) * (tt.abs() @ wl.abs().t() + bl.abs())
    assert ((gb - gb_ref).abs() <= gb_bound).all(), "timbre_linear"
    ref, bound, outs_oracle = _fp64_reference(sd, codes, timbre, gb)
    got = dict(outs=outs, zp=parts[0], zc=parts[1], zr=parts[2])
    for k in ("zp", "zc", "zr", "outs"):
        e = (got[k].cpu().double() - ref[k]).abs()
        assert (e <= bound[k]).all(), f"{k}: max err {e.max():.3e}, max err / bound {(e / bound[k].clamp_min(1e-300)).max():.2f}"
    if n_r == 0:
        assert torch.equal(parts[2].cpu(), torch.zeros(B, 1024, T)), "z_r must be zeros without residual codes"
    # and the whole thing against the oracle's own fp64 gamma | beta
    assert float((outs.cpu().double() - outs_oracle).abs().max()) <= 1e-4
    print(f"n_c={n_c} n_r={n_r} T={T}: outs max err {float((outs.cpu().double() - ref['outs']).abs().max()):.2e} "
          f"(bound median {float(bound['outs'].median()):.2e}, u = {U:.2e})")


@pytest.mark.gpu
def test_dequantize_out_of_range_code_gives_nan_in_its_frame_only(built_lib):
    m = _model(0)
    sd = state_dicts(0)["quantizer"]
    B, T = 2, 9
    codes = _random_codes(B, T, 2, 3, seed=5)
    timbre = (0.3 * torch.randn(B, 1024, generator=torch.Generator().manual_seed(6))).cuda()
    bad = [c.clone() for c in codes]
    bad[1][1, 1, 4] = 1024                       # utterance 1, frame 4, second content row
    gb = torch.full((B, 2048), float("nan"), device="cuda")
    outs, _ = _dequantize_raw(m, bad, timbre, False, gb_tap=gb)
    ref, bound, _ = _fp64_reference(sd, codes, timbre, gb.cpu().double())
    nan = torch.isnan(outs.cpu())
    frame = torch.zeros(B, 1024, T, dtype=torch.bool)
    frame[1, :, 4] = True
    assert torch.equal(nan, frame), "exactly the frame with the out-of-range code is NaN"
    e = (outs.cpu().double() - ref["outs"]).abs()
    assert (e[~frame] <= bound["outs"][~frame]).all()


@pytest.mark.gpu
def test_invalid_arguments(built_lib):
    import facodec_b200 as fb
    m = _model(0)
    codec = fb.Codec(m)
    B, T = 2, 7
    cp, cc, cr = _random_codes(B, T, 2, 3, seed=9)
    tb = torch.zeros(B, 1024, device="cuda")
    for codes, timbre in (([cp, torch.cat([cc, cc[:, :1]], 1), cr], tb), ([cp, cc, torch.cat([cr, cr[:, :1]], 1)], tb),
                          ([cp, cc[:1], cr], tb), ([cp, cc, cr[:, :, :5]], tb), ([cp, cc, cr], tb[:, :1000]),
                          ([cp, cc, cr], tb[:1])):
        with pytest.raises(ValueError):
            codec.decode(codes, timbre)
        with pytest.raises(ValueError):
            m.quantizer.from_codes(codes, timbre)
    with pytest.raises(fb.FacError):
        codec.decode([cp.cpu(), cc, cr], tb)
    with pytest.raises(fb.FacError):
        codec.decode([cp, cc, cr], tb.cpu())
    for v in (-1, 1024):
        c2 = cr.clone()
        c2[0, 2, 3] = v
        with pytest.raises(IndexError):
            codec.decode([cp, cc, c2], tb)
    # the C-ABI rejects bad row counts and a missing residual tensor with FAC_ERR_INVALID
    e = m.quantizer._engine
    y = torch.empty(B, 1, 300 * T, device="cuda")
    for n_c_rows, r_ptr, n_r_rows in ((3, cr, 3), (0, cr, 3), (2, cr, 4), (2, None, 1), (2, cr, -1)):
        rc = e.L.fac_codes_decode(e.handle, _p(cp), _p(cc), n_c_rows, _p(r_ptr), n_r_rows, _p(tb), B, T, _p(y), None)
        assert rc == -1, (n_c_rows, n_r_rows)
    assert e.L.fac_codes_decode(e.handle, _p(cp), _p(cc), 2, _p(cr), 3, _p(tb), B, 0, _p(y), None) == -1
    assert e.L.fac_codes_decode(e.handle, _p(cp), _p(cc), 2, _p(cr), 3, None, B, T, _p(y), None) == -1


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_decode_golden_codes(name, built_lib):
    import facodec_b200 as fb
    c = GOLDEN_CASES[name]
    g = load_golden(name)
    codec = fb.Codec(_model(c["wseed"]))
    codes = [torch.from_numpy(g[k]).cuda() for k in ("codes_p", "codes_c", "codes_r")]
    y = codec.decode(codes, torch.from_numpy(g["timbre"]).cuda())
    assert tuple(y.shape) == g["y"].shape
    e = _rms(y, g["y"])
    print(f"{name}: decode(golden codes) vs golden y rms {e:.3g}")
    assert e <= RMS_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("name", PIN_CASES)
def test_decode_pinned_codes(name, built_lib):
    import facodec_b200 as fb
    c = _pin_case(_pin("from_codes"), name)
    m = _model(1)
    codes = [c[k].cuda() for k in ("codes_p", "codes_c", "codes_r")]
    y = fb.Codec(m).decode(codes, c["timbre"].cuda())
    assert tuple(y.shape) == tuple(c["y"].shape)
    assert _rms(y, c["y"]) <= RMS_TOL
    outs, parts = m.quantizer.from_codes(codes, c["timbre"].cuda())
    assert float((outs.cpu() - c["outs"]).abs().max()) <= 2e-4      # AdaLN output, |outs| ~ 1 (as test_gpu_parity)
    for k, t in zip(("z_p", "z_c", "z_r"), parts):
        assert float((t.cpu() - c[k]).abs().max()) <= 1e-5 * max(1.0, float(c[k].abs().max())), k


@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(32, 96000), (3, 12345)])
def test_encode_then_decode_equals_forward(B, T, built_lib):
    import facodec_b200 as fb
    from facodec_b200 import synth
    codec = fb.Codec(_model(0))
    x = synth.synth_waves(B, T, seed=114514 if B == 32 else 31).cuda()
    y, codes_f, timbre_f = codec.forward(x)
    codes, timbre = codec.encode(x)
    for a, b in zip(codes, codes_f):
        assert a.dtype == torch.int64 and torch.equal(a, b)
    assert torch.equal(timbre, timbre_f)
    y2 = codec.decode(codes, timbre)
    torch.cuda.synchronize()
    assert y2.shape == y.shape
    e = _rms(y2, y)
    print(f"B={B} T={T}: decode(encode(x)) vs forward(x) y rms {e:.3g} (signal rms {float(y.double().pow(2).mean().sqrt()):.3g}), "
          f"bit-equal {bool(torch.equal(y2, y))}")
    assert e <= RMS_TOL


@pytest.mark.gpu
def test_decode_with_another_timbre(built_lib):
    """Codes of b2_t7200 decoded with the timbre of b2_t6000_fullwaves, against the CPU oracle."""
    import facodec_b200 as fb
    g = load_golden("b2_t7200")
    other = torch.from_numpy(load_golden("b2_t6000_fullwaves")["timbre"])
    sds = state_dicts(0)
    codes = [torch.from_numpy(g[k]) for k in ("codes_p", "codes_c", "codes_r")]
    codec = fb.Codec(_model(0))
    y_swap = codec.decode([c.cuda() for c in codes], other.cuda())
    y_own = codec.decode([c.cuda() for c in codes], torch.from_numpy(g["timbre"]).cuda())
    with torch.no_grad():
        y_ref = O.decoder_forward(sds["decoder"], FC.quantizer_from_codes(sds["quantizer"], *codes, other)[0])
    e, d = _rms(y_swap, y_ref), _rms(y_swap, y_own)
    print(f"timbre swap: vs oracle rms {e:.3g}, distance from own timbre rms {d:.3g}")
    assert e <= RMS_TOL
    assert d > 20 * RMS_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", [[3000, 300, 9000, 24000, 600], [30000], [4500, 1500]])
def test_stream_decode_codes_equals_offline(sizes, built_lib):
    import facodec_b200 as fb
    from test_gpu_stream import chunks_of
    m = _model(1)
    g = torch.Generator().manual_seed(77)
    B, T = 3, 60000
    x = (torch.randn(B, 1, T, generator=g) * 0.1).cuda()
    codec = fb.Codec(m)
    codes, timbre = codec.encode(x)
    codes[2] = codes[2][:, :2]                   # two residual rows: the row count reaches the stream too
    y_off = codec.decode(codes, timbre)
    with fb.CodecStream(m, B) as s:
        ys = [s.decode_codes([c[:, :, p // 300:(p + n) // 300] for c in codes], timbre) for p, n in chunks_of(T, sizes)]
    y_st = torch.cat(ys, dim=2)
    torch.cuda.synchronize()
    assert y_st.shape == y_off.shape
    e = _rms(y_st, y_off)
    print(f"stream decode_codes vs offline decode: rms {e:.3g} bit-equal {bool(torch.equal(y_st, y_off))}")
    assert e <= RMS_TOL


@pytest.mark.gpu
def test_stream_decode_codes_errors(built_lib):
    import facodec_b200 as fb
    m = _model(1)
    cp, cc, cr = _random_codes(1, 12, 2, 3, seed=3)
    tb = torch.zeros(1, 1024, device="cuda")
    with fb.CodecStream(m, 1) as s:
        with pytest.raises(fb.FacError):
            s.decode_codes([c[:, :, :4] for c in (cp, cc, cr)], tb)          # first chunk < 10 frames
        with pytest.raises(ValueError):
            s.decode_codes([c.repeat(2, 1, 1) for c in (cp, cc, cr)], tb.repeat(2, 1))   # batch differs from the stream's
        with pytest.raises(fb.FacError):
            s.decode_codes([cp, cc, cr], tb.cpu())
        with pytest.raises(IndexError):
            s.decode_codes([cp, cc, cr.clone().fill_(1024)], tb)


@pytest.mark.gpu
def test_dac_file_round_trip_decodes_identically(tmp_path, built_lib):
    import facodec_b200 as fb
    from facodec_b200 import codefile, synth
    codec = fb.Codec(_model(0))
    x = synth.synth_waves(2, 7000, seed=7).cuda()
    for n_c in (1, 2):
        codes, timbre = codec.encode(x, n_c=n_c)
        path = codefile.from_forward(codes, original_length=x.shape[-1]).save(tmp_path / f"utt{n_c}")
        back = [c.cuda() for c in codefile.DACFile.load(path).unpack()]
        assert torch.equal(codec.decode(back, timbre), codec.decode(codes, timbre))
