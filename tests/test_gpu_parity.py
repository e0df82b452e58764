"""GPU parity tests proper: the CUDA path, called through the C-ABI (via the thin ctypes module
shim), against (a) the committed golden fixtures made from the imported unmodified reference,
(b) the oracle restatement run live on this box's CPU, (c) size-independent properties at
BASELINE configs[1] size (B=32 x 4 s).

Bars (BASELINE.json north_star): VQ code indices bit-exact; waveform RMS error <= 1e-4.
Float tensors upstream of the VQ are compared with tolerances stated inline.
"""
import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, case_inputs, load_golden, state_dicts

pytestmark = pytest.mark.gpu

RMS_TOL = 1e-4          # north_star: reconstructed waveform within 1e-4 RMS
Z_RTOL = 2e-5           # encoder latents: max |dz| <= Z_RTOL * max |z| (fp32 re-association only)


def rms(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float(((a - b) ** 2).mean().sqrt())


_MODEL = {}


def model_for(seed):
    import facodec_b200 as fb
    if seed not in _MODEL:
        _MODEL.clear()
        m = fb.build_model()
        sds = state_dicts(seed)
        for k in ("encoder", "quantizer", "decoder"):
            m[k].load_state_dict(sds[k])
            m[k].eval()
        _MODEL[seed] = m
    return _MODEL[seed]


def run_model(m, x, n_c, kw):
    dev = torch.device("cuda:0")
    xd = x.to(dev)
    kwd = {k: v.to(dev) for k, v in kw.items()}
    z = m.encoder(xd)
    q = m.quantizer(z, xd, n_c=n_c, return_codes=True, **kwd)
    y = m.decoder(q[0])
    torch.cuda.synchronize()
    return z, q, y


@pytest.mark.parametrize("name", ["b2_t7200", "b1_t7000_ragged", "b3_t1500_short", "b2_t6000_fullwaves", "b1_t96000"])
def test_golden_end_to_end(name, built_lib):
    c = GOLDEN_CASES[name]
    g = load_golden(name)
    m = model_for(c["wseed"])
    x, kw = case_inputs(c)
    z, q, y = run_model(m, x, c["n_c"], kw)
    assert tuple(z.shape) == g["z"].shape and tuple(y.shape) == g["y"].shape
    zerr = np.abs(z.cpu().numpy() - g["z"]).max()
    assert zerr <= Z_RTOL * np.abs(g["z"]).max(), f"z max err {zerr}"
    for k, t in zip(("codes_p", "codes_c", "codes_r"), q[5]):
        assert t.dtype == torch.int64 and tuple(t.shape) == g[k].shape
        assert np.array_equal(t.cpu().numpy(), g[k]), f"{k}: {(t.cpu().numpy() != g[k]).sum()} indices differ"
    assert np.abs(q[4].cpu().numpy() - g["timbre"]).max() <= 1e-5 * max(1.0, np.abs(g["timbre"]).max())
    assert np.abs(q[0].cpu().numpy() - g["outs"]).max() <= 2e-4       # AdaLN output, |outs| ~ 1
    assert abs(float(q[2]) - float(g["commitment"])) <= 1e-5 * abs(float(g["commitment"]))
    assert abs(float(q[3]) - float(g["codebook"])) <= 1e-5 * abs(float(g["codebook"]))
    if "z_p" in g:
        for k, t in zip(("z_p", "z_c", "z_r"), q[1]):
            assert np.abs(t.cpu().numpy() - g[k]).max() <= 1e-5 * max(1.0, np.abs(g[k]).max()), k
    e = rms(y, g["y"])
    assert e <= RMS_TOL, f"waveform RMS error {e}"
    assert float(y.abs().max()) < 1.0


@pytest.mark.parametrize("name", ["b2_t7200", "b3_t1500_short"])
def test_golden_teacher_forced_stages(name, built_lib):
    """Each module on the reference's own inputs (isolates the three entry points)."""
    c = GOLDEN_CASES[name]
    g = load_golden(name)
    m = model_for(c["wseed"])
    x, kw = case_inputs(c)
    dev = torch.device("cuda:0")
    zg = torch.from_numpy(g["z"]).to(dev)
    q = m.quantizer(zg, x.to(dev), n_c=c["n_c"], return_codes=True)
    for k, t in zip(("codes_p", "codes_c", "codes_r"), q[5]):
        assert np.array_equal(t.cpu().numpy(), g[k]), k
    y = m.decoder(torch.from_numpy(g["outs"]).to(dev))
    assert rms(y, g["y"]) <= RMS_TOL


def test_live_oracle_new_seed(built_lib):
    """Fresh weights + waves, oracle run on this box's CPU."""
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    seed = 5
    sds = state_dicts(seed)
    m = model_for(seed)
    x = synth.synth_waves(2, 9000, seed=77)
    zo, qo, yo = O.codec_forward(sds, x, n_c=2)
    z, q, y = run_model(m, x, 2, {})
    assert (z.cpu() - zo).abs().max() <= Z_RTOL * zo.abs().max()
    for a, b in zip(q[5], qo[5]):
        assert torch.equal(a.cpu(), b)
    assert rms(y, yo) <= RMS_TOL


@pytest.mark.parametrize("B,T,n_c", [(35, 4500, 2), (1, 1030, 2), (2, 2999, 1), (3, 12345, 2)])
def test_live_oracle_odd_shapes(B, T, n_c, built_lib):
    """Shapes the fixtures do not hold, against the oracle run on this box's CPU: more than 32 utterances (the LSTM takes 32
    sequences per launch), the shortest length the quantizer's centred STFT accepts (+ ragged), lengths that are not
    multiples of the 300-sample hop or of any tile size."""
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    sds = state_dicts(0)
    m = model_for(0)
    x = synth.synth_waves(B, T, seed=1000 + B + T)
    torch.set_num_threads(max(1, min(16, len(__import__("os").sched_getaffinity(0)))))
    zo, qo, yo = O.codec_forward(sds, x, n_c=n_c)
    z, q, y = run_model(m, x, n_c, {})
    assert z.shape == zo.shape and y.shape == yo.shape
    assert (z.cpu() - zo).abs().max() <= Z_RTOL * zo.abs().max()
    for a, b in zip(q[5], qo[5]):
        assert torch.equal(a.cpu(), b), f"{int((a.cpu() != b).sum())} of {b.numel()} indices differ"
    assert rms(y, yo) <= RMS_TOL


def test_fused_codec_forward_equals_three_calls(built_lib):
    import facodec_b200 as fb
    from facodec_b200 import synth
    m = model_for(0)
    x = synth.synth_waves(3, 6000, seed=4).cuda()
    z, q, y = run_model(m, x.cpu(), 2, {})
    codec = fb.Codec(m)
    y2, codes2, timbre2 = codec.forward(x, n_c=2)
    torch.cuda.synchronize()
    assert torch.equal(y, y2)
    for a, b in zip(q[5], codes2):
        assert torch.equal(a, b)
    assert torch.equal(q[4], timbre2)
    yh, codes_h = codec.forward_host(x.cpu().contiguous(), n_c=2)
    assert torch.equal(yh, y.cpu())
    for a, b in zip(q[5], codes_h):
        assert torch.equal(a.cpu(), b)
    assert codec.launch_count() > 50


def test_cuda_graph_replay_equals_eager(built_lib):
    """Codec.forward_graphed: the whole forward (cooperative LSTM launches, the forked quantizer front) captured once and
    replayed -- same bits as the eager call, also for a second input of the same shape and after another shape was used."""
    import facodec_b200 as fb
    from facodec_b200 import synth
    m = model_for(0)
    codec = fb.Codec(m)
    xa = synth.synth_waves(1, 24000, seed=21).cuda()
    xb = synth.synth_waves(1, 24000, seed=22).cuda()
    xc = synth.synth_waves(2, 6000, seed=23).cuda()
    for x in (xa, xc, xb, xa):
        y, codes, timbre = codec.forward(x, n_c=2)
        yg, codes_g, timbre_g = codec.forward_graphed(x, n_c=2)
        torch.cuda.synchronize()
        assert torch.equal(y, yg) and torch.equal(timbre, timbre_g)
        for a, b in zip(codes, codes_g):
            assert torch.equal(a, b)
    assert len(codec._graphs) == 2


def test_full_size_properties(built_lib):
    """BASELINE configs[1]: B=32 x 4 s.  (1) utterance 0 == golden b1_t96000 (same PseudoDataset
    stream); (2) batch invariance: an utterance decodes to the same bits alone or inside the batch;
    (3) range/shape invariants."""
    import facodec_b200 as fb
    from facodec_b200 import synth
    m = model_for(0)
    codec = fb.Codec(m)
    x = synth.synth_waves(32, 96000).cuda()
    y, codes, timbre = codec.forward(x, n_c=2)
    torch.cuda.synchronize()
    assert tuple(y.shape) == (32, 1, 96000)
    assert torch.isfinite(y).all() and float(y.abs().max()) < 1.0
    for c_, n in zip(codes, (1, 2, 3)):
        assert tuple(c_.shape) == (32, n, 320) and int(c_.min()) >= 0 and int(c_.max()) < 1024
    g = load_golden("b1_t96000")
    assert np.array_equal(codes[0][0].cpu().numpy(), g["codes_p"][0])
    assert np.array_equal(codes[1][0].cpu().numpy(), g["codes_c"][0])
    assert np.array_equal(codes[2][0].cpu().numpy(), g["codes_r"][0])
    assert rms(y[0], g["y"][0]) <= RMS_TOL
    for i in (0, 17, 31):
        yi, ci, ti = codec.forward(x[i:i + 1].contiguous(), n_c=2)
        assert torch.equal(yi[0], y[i]), f"utterance {i}: batch-dependent result"
        for a, b in zip(ci, codes):
            assert torch.equal(a[0], b[i])


def test_rvq_against_oracle_and_properties(built_lib):
    """quantize/rvq.py ResidualVQ (BASELINE configs[3] geometry: 4 x 1024 entries, 1024 -> 8)."""
    import facodec_b200 as fb
    from oracle import facodec_oracle as O
    rvq = fb.ResidualVQ(num_quantizers=4, codebook_size=10, dim=1024, codebook_dim=8, commitment=0.25).eval()
    g = torch.Generator().manual_seed(11)
    x = torch.randn(3, 1024, 41, generator=g)
    layers = []
    for i in range(4):
        layers.append(dict(in_w=rvq._folded(i, "in_proj"), in_b=rvq._p[f"layers/{i}/in_proj/bias"].detach(),
                           out_w=rvq._folded(i, "out_proj"), out_b=rvq._p[f"layers/{i}/out_proj/bias"].detach(),
                           codebook=rvq._p[f"layers/{i}/_codebook/weight"].detach()))
    with torch.no_grad():
        qo, io, lo, ao = O.fvq_residual_vq(layers, x)
    q, idx, loss, allq = rvq(x.cuda())
    assert torch.equal(idx.cpu(), io)
    assert (q.cpu() - qo).abs().max() <= 1e-5 and (allq.cpu() - ao).abs().max() <= 1e-5
    assert float(loss.abs().sum()) == 0.0
    # larger, channels-last, properties: quantized_out == sum of stages; indices in range
    xb = torch.randn(64, 256, 1024, generator=g).cuda()
    q2, idx2, _, allq2 = rvq(xb, channels_last=True)
    assert int(idx2.min()) >= 0 and int(idx2.max()) < 1024
    assert (allq2.sum(0) - q2).abs().max() <= 1e-5
    q3, idx3, _, _ = rvq(xb.transpose(1, 2).contiguous())
    assert torch.equal(idx3, idx2) and torch.equal(q3.transpose(1, 2), q2)


def test_alias_free_activation(built_lib):
    import facodec_b200 as fb
    from oracle import facodec_oracle as O
    g = torch.Generator().manual_seed(2)
    for (B, C, T) in ((2, 5, 50), (1, 3, 700), (2, 2, 1)):
        x = torch.randn(B, C, T, generator=g)
        ident = fb.Activation1d(identity=True)
        y = ident(x.cuda()).cpu()
        assert (y - O.alias_free_act(x, lambda u: u)).abs().max() <= 2e-6
        act = fb.Activation1d(C, alpha_logscale=True)
        with torch.no_grad():
            act.alpha.copy_(torch.randn(C, generator=g) * 0.3)
            act.beta.copy_(torch.randn(C, generator=g) * 0.3)
        a, b = torch.exp(act.alpha).view(1, C, 1), torch.exp(act.beta).view(1, C, 1)
        ref = O.alias_free_act(x, lambda u: u + (1.0 / (b + 1e-9)) * torch.sin(u * a).pow(2))
        assert (act(x.cuda()).cpu() - ref).abs().max() <= 5e-6


def test_error_paths(built_lib):
    import facodec_b200 as fb
    m = model_for(0)
    with pytest.raises(fb.FacError):
        m.encoder(torch.zeros(1, 1, 3000))                       # CPU tensor: no fallback
    with pytest.raises(fb.FacError):
        m.quantizer(torch.zeros(1, 1024, 2).cuda(), torch.zeros(1, 1, 600).cuda())   # shorter than STFT padding


@pytest.mark.parametrize("mode", [0, 1])
def test_other_precision_modes_keep_parity(mode, built_lib):
    """fac_set_option("tensor_cores", 0 | 1): the fp32 FMA path and the decoder-only tensor-core path
    stay correct (default mode 2 is what every other test runs)."""
    c = GOLDEN_CASES["b2_t7200"]
    g = load_golden("b2_t7200")
    m = model_for(c["wseed"])
    eng = m.encoder._engine
    x, kw = case_inputs(c)
    try:
        eng.set_option("tensor_cores", mode, torch.device("cuda:0"))
        z, q, y = run_model(m, x, c["n_c"], kw)
    finally:
        eng.set_option("tensor_cores", 2, torch.device("cuda:0"))
    for k, t in zip(("codes_p", "codes_c", "codes_r"), q[5]):
        assert np.array_equal(t.cpu().numpy(), g[k]), k
    assert np.abs(z.cpu().numpy() - g["z"]).max() <= Z_RTOL * np.abs(g["z"]).max()
    assert rms(y, g["y"]) <= (5e-7 if mode == 0 else RMS_TOL)


def test_encoder_f16x2_option_keeps_parity(built_lib):
    """fac_set_option("encoder_f16x2", 0 | 1): the promoted kernel with the TF32 pair instead of the default fp16 hi +
    2^11-scaled lo split (22 mantissa bits either way).  Codes stay bit-exact on the fixtures with either."""
    for name in ("b2_t7200", "b1_t96000"):
        c = GOLDEN_CASES[name]
        g = load_golden(name)
        m = model_for(c["wseed"])
        eng = m.encoder._engine
        x, kw = case_inputs(c)
        try:
            eng.set_option("encoder_f16x2", 0, torch.device("cuda:0"))
            z, q, y = run_model(m, x, c["n_c"], kw)
        finally:
            eng.set_option("encoder_f16x2", 1, torch.device("cuda:0"))
        for k, t in zip(("codes_p", "codes_c", "codes_r"), q[5]):
            assert np.array_equal(t.cpu().numpy(), g[k]), k
        assert np.abs(z.cpu().numpy() - g["z"]).max() <= Z_RTOL * np.abs(g["z"]).max()
        assert rms(y, g["y"]) <= RMS_TOL


# ---------------------------------------------------------------------------------------------------------------
# round 2: voice conversion (modules/redecoder.py + the non-causal, LSTM-free decoder; reconstruct_redecoder.py:108-122)
# ---------------------------------------------------------------------------------------------------------------
_REDEC = {}


def redec_model_for(seed):
    import facodec_b200 as fb
    from facodec_b200 import synth
    if seed not in _REDEC:
        _REDEC.clear()
        m = fb.build_model(stage="redecoder")
        sds = synth.synth_redecoder_state_dicts(seed)
        for k in ("encoder", "decoder"):
            m[k].load_state_dict(sds[k])
            m[k].eval()
        _REDEC[seed] = m
    return _REDEC[seed]


@pytest.mark.parametrize("name", ["redec_b2_t7200_vc", "redec_b2_t7200_full", "redec_b3_t1500_short"])
def test_redecoder_golden(name, built_lib):
    """Fixtures made from the imported reference (oracle/make_golden.py redecoder): codes + timbre of a codec fixture ->
    redecoder.encoder -> redecoder.decoder.  z within fp32-class tolerance, waveform RMS <= 1e-4; the fused
    fac_voice_convert call gives the same bits as the two-call surface."""
    import facodec_b200 as fb
    from conftest import REDEC_CASES
    c = REDEC_CASES[name]
    g = load_golden(name)
    src = load_golden(c["src"])
    m = redec_model_for(c["wseed"])
    dev = torch.device("cuda:0")
    cp, cc, timbre = (torch.from_numpy(src[k]).to(dev) for k in ("codes_p", "codes_c", "timbre"))
    z = m.encoder(cp, cc, timbre, use_p_code=c["use_p"], n_c=c["n_c"])
    y = m.decoder(z)
    torch.cuda.synchronize()
    assert tuple(z.shape) == g["z"].shape and tuple(y.shape) == g["y"].shape
    zerr = np.abs(z.cpu().numpy() - g["z"]).max()
    assert zerr <= 2e-4 * max(1.0, np.abs(g["z"]).max()), f"z max err {zerr}"          # bf16 hi/lo class (16 mantissa bits)
    assert rms(y, g["y"]) <= RMS_TOL
    # teacher-forced decoder on the reference's own z
    assert rms(m.decoder(torch.from_numpy(g["z"]).to(dev)), g["y"]) <= RMS_TOL
    y2 = fb.VoiceConverter(m).convert([cp, cc], timbre, use_p_code=c["use_p"], n_c=c["n_c"])
    torch.cuda.synchronize()
    assert torch.equal(y2, y)


def test_voice_conversion_flow_vs_live_oracle(built_lib):
    """reconstruct_redecoder.py:108-122 end to end on this box: codec encode of a source and a reference utterance, then
    model.encoder(codes[0], codes[1], timbre_of_reference, use_p_code=False, n_c=1) -> model.decoder, against the oracle."""
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    codec = model_for(0)
    sds = state_dicts(0)
    rm = redec_model_for(0)
    rsds = synth.synth_redecoder_state_dicts(0)
    src = synth.synth_waves(1, 9000, seed=41)
    ref = synth.synth_waves(1, 6000, seed=42)
    dev = torch.device("cuda:0")
    _, q, _ = run_model(codec, src, 2, {})
    _, q2, _ = run_model(codec, ref, 2, {})
    y = rm.decoder(rm.encoder(q[5][0], q[5][1], q2[4], use_p_code=False, n_c=1))
    torch.cuda.synchronize()
    _, qo, _ = O.codec_forward(sds, src, n_c=2)
    _, qo2, _ = O.codec_forward(sds, ref, n_c=2)
    zo, yo = O.voice_convert(rsds, qo[5], qo2[4])
    assert torch.equal(q[5][0].cpu(), qo[5][0]) and torch.equal(q[5][1].cpu(), qo[5][1])
    assert rms(y, yo) <= RMS_TOL
    with pytest.raises(IndexError):
        rm.encoder(q[5][0], q[5][1][:, :1], q2[4], n_c=2)
    import facodec_b200 as fb
    with pytest.raises(fb.FacError):
        rm.encoder(q[5][0], q[5][1].cpu(), q2[4])                    # input on another device: no silent foreign pointer


@pytest.mark.parametrize("indim,outdim,heads,glob,T", [(1024, 1, 2, False, 320), (64, 1024, 1, False, 77), (256, 400, 1, True, 50)])
def test_cnnlstm_predictor_heads_vs_oracle(indim, outdim, heads, glob, T, built_lib):
    """modules/quantize.py:106-125 CNNLSTM forward (FApredictors f0 / phone / timbre head geometries, scaled): alias-free
    SnakeBeta + conv stacks + Linear heads against the oracle (pinned bit-for-bit to the imported class in test_oracle.py).
    Tolerance: decoder-class precision (bf16 hi/lo operands), 2e-3 of the output scale."""
    import facodec_b200 as fb
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    m = fb.CNNLSTM(indim, outdim, heads, global_pred=glob).eval()
    sd = synth.synth_cnnlstm(11, indim, outdim, heads)
    m.load_state_dict(sd)
    assert set(sd) <= set(m.state_dict()) and any(k.endswith("upsample.filter") for k in m.state_dict())
    g = torch.Generator().manual_seed(indim + T)
    x = torch.randn(3, indim, T, generator=g)
    with torch.no_grad():
        ref = O.cnnlstm_forward(sd, x, heads, global_pred=glob)
    out = m(x.cuda())
    torch.cuda.synchronize()
    assert len(out) == heads
    for a, b in zip(out, ref):
        assert tuple(a.shape) == tuple(b.shape)
        err = float((a.cpu() - b).abs().max())
        assert err <= 2e-3 * max(1.0, float(b.abs().max())), f"max err {err}"


@pytest.mark.parametrize("timbre_norm", [True, False])
def test_fa_predictors_vs_oracle(timbre_norm, built_lib):
    """modules/quantize.py:456-619 FApredictors with build_model's flags (modules/commons.py:311-322), both forward variants,
    in_dim 64 (the head widths 1 / 1024 / 20000 are the reference's): every prediction against the oracle (pinned to the
    imported class in test_oracle.py).  Tolerance: decoder-class precision (bf16 hi/lo operands), 2e-3 of the output scale."""
    import facodec_b200 as fb
    from oracle import facodec_oracle as O
    flags = dict(use_gr_content_f0=False, use_gr_prosody_phone=False, use_gr_residual_f0=True, use_gr_residual_phone=True,
                 use_gr_timbre_content=True, use_gr_timbre_prosody=False, use_gr_x_timbre=True, norm_f0=True)
    m = fb.FApredictors(in_dim=64, timbre_norm=timbre_norm, use_gr_content_global_f0=True, **flags).eval()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    assert "rev_f0_predictor.1.model.0.block.1.weight_g" in sd and "rev_timbre_predictor.1.heads.0.weight" in sd
    assert ("timbre_predictor.weight" in sd) == timbre_norm and ("global_f0_predictor.bias" in sd) == timbre_norm
    m.load_state_dict(sd)
    g = torch.Generator().manual_seed(8)
    lat = [torch.randn(2, 64, 41, generator=g) for _ in range(3 if timbre_norm else 4)]
    timbre = torch.randn(2, 64, generator=g)
    with torch.no_grad():
        ref = O.fa_predictors_forward(sd, lat, timbre if timbre_norm else None, timbre_norm=timbre_norm, **flags)
    if timbre_norm:
        got = m([t.cuda() for t in lat], timbre.cuda())
    else:
        got = m([t.cuda() for t in lat])
    torch.cuda.synchronize()
    for a, b in zip(got, ref):
        assert a.keys() == b.keys()
        for k in a:
            assert tuple(a[k].shape) == tuple(b[k].shape), k
            err = float((a[k].cpu() - b[k]).abs().max())
            assert err <= 2e-3 * max(1.0, float(b[k].abs().max())), f"{k}: max err {err}"
    with pytest.raises(fb.FacError):
        m([t for t in lat], timbre) if timbre_norm else m([t for t in lat])          # CPU tensors: no fallback


def test_dataset_mel_vs_oracle(built_lib):
    """meldataset.py:37-47 (16 kHz-default filterbank, centre=True frames) through fac_dataset_mel against the oracle
    restatement (pinned to the imported meldataset module in test_oracle.py).  Log-mel values are O(1): 2e-4 absolute."""
    from facodec_b200 import meldataset as MD
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    fb = synth.melscale_fbanks_htk(sample_rate=16000, f_max=8000.0)
    win = synth.hann_window_periodic(1200)
    for (B, T) in ((2, 7200), (1, 24001), (3, 1500)):
        w = synth.synth_waves(B, T, seed=T)[:, 0]
        ref = O.dataset_mel(w, win, fb)
        got = MD.to_mel_batch(w.cuda()).cpu()
        assert tuple(got.shape) == tuple(ref.shape) == (B, 80, T // 300 + 1)
        assert float((got - ref).abs().max()) <= 2e-4
    one = MD.preprocess(synth.synth_waves(1, 3000, seed=1)[0, 0].numpy())
    assert tuple(one.shape) == (1, 80, 11)
    wave, mel = MD.PseudoDataset(range=(1, 2))[0]
    assert mel.shape[0] == 80 and mel.shape[1] == wave.shape[0] // 300 + 1


def test_two_handles_on_two_devices_in_one_process(built_lib):
    """Launch configuration (> 48 KB dynamic shared-memory opt-in, SM count) is per device: a second engine on cuda:1 in the
    same process must work and give the same bits as cuda:0 (round-1 ADVICE: process-wide statics broke this)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import facodec_b200 as fb
    from facodec_b200 import synth
    sds = state_dicts(0)
    x = synth.synth_waves(2, 9000, seed=8)
    outs = []
    for d in (0, 1):
        m = fb.build_model()
        for k in ("encoder", "quantizer", "decoder"):
            m[k].load_state_dict(sds[k])
            m[k].eval()
        dev = torch.device("cuda", d)
        xd = x.to(dev)
        z = m.encoder(xd)
        q = m.quantizer(z, xd, n_c=2, return_codes=True)
        y = m.decoder(q[0])
        torch.cuda.synchronize(dev)
        outs.append((y.cpu(), [c.cpu() for c in q[5]]))
        with pytest.raises(fb.FacError):
            m.encoder(x.to(torch.device("cuda", 1 - d)))          # engine is bound to its device
    assert torch.equal(outs[0][0], outs[1][0])
    for a, b in zip(outs[0][1], outs[1][1]):
        assert torch.equal(a, b)
