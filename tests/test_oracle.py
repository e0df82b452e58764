"""CPU: the oracle restatement against the committed golden fixtures generated from the imported unmodified
reference (oracle/make_golden.py): whole-model cases (tests/golden/<case>.npz) and the module-level pins
(tests/golden/pin_*.npz)."""
import hashlib
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, case_inputs, load_golden, state_dicts
from oracle import facodec_oracle as O
from oracle import ref_import

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Bit-exact where the fixtures were made (same CPU, same ATen kernels); on another host CPU oneDNN may pick
# other kernels, so floats get a tight tolerance there.
SAME_HOST = ref_import.available()
ATOL = 0.0 if SAME_HOST else 2e-5


def _pin(name):
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "pin_" + name + ".npz")))


def _pinned_params(pin, seed):
    """The seeded parameters (oracle/make_golden.py seeded_params) and stored buffers the pinned module ran with."""
    from oracle import make_golden
    shapes = {k[len("shape/"):]: v for k, v in pin.items() if k.startswith("shape/")}
    sd = make_golden.seeded_params(shapes, seed)
    sd.update({k[len("buffer/"):]: torch.from_numpy(v) for k, v in pin.items() if k.startswith("buffer/")})
    return sd


def _close(a, b, name):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, name
    if ATOL == 0.0:
        assert np.array_equal(a, b), f"{name}: max diff {np.abs(a - b).max()}"
    else:
        assert np.abs(a - b).max() <= ATOL * max(1.0, np.abs(b).max()), name


def test_case_table():
    from oracle import make_golden
    assert make_golden.CASES == GOLDEN_CASES
    for name in GOLDEN_CASES:
        assert os.path.exists(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))


def test_synth_is_host_independent():
    """Synthetic checkpoints must be the same bits everywhere (golden fixtures depend on it)."""
    from facodec_b200 import synth
    sd = synth.synth_encoder(1)
    h = hashlib.sha256()
    for k in ("block.0.conv.conv.weight_g", "block.1.block.0.block.1.conv.conv.weight_v", "block.6.alpha"):
        h.update(sd[k].numpy().tobytes())
    assert h.hexdigest() == "db65aa08d774396d996e318b9407e70d4417e942368011e08c72c2d351e27314"
    w = synth.synth_waves(1, 1000, seed=3)
    assert abs(float(w.abs().max()) - 1.0) < 1e-7


@pytest.mark.parametrize("name", ["b2_t7200", "b1_t7000_ragged", "b3_t1500_short", "b2_t6000_fullwaves", "b1_t96000"])
def test_oracle_matches_golden(name):
    c = GOLDEN_CASES[name]
    g = load_golden(name)
    sds = state_dicts(c["wseed"])
    x, kw = case_inputs(c)
    with torch.no_grad():
        z = O.encoder_forward(sds["encoder"], x)
        q = O.quantizer_forward(sds["quantizer"], z, x, n_c=c["n_c"], return_codes=True, **kw)
        y = O.decoder_forward(sds["decoder"], q[0])
    _close(z, g["z"], "z")
    _close(q[0], g["outs"], "outs")
    _close(q[4], g["timbre"], "timbre")
    _close(y, g["y"], "y")
    for k, t in zip(("codes_p", "codes_c", "codes_r"), q[5]):
        if SAME_HOST:
            assert np.array_equal(t.numpy(), g[k]), k
        else:
            assert (t.numpy() != g[k]).mean() < 0.02, k
    assert abs(float(q[2]) - float(g["commitment"])) <= 1e-5 * abs(float(g["commitment"]))
    if "z_p" in g:
        for k, t in zip(("z_p", "z_c", "z_r"), q[1]):
            _close(t, g[k], k)


def test_oracle_matches_imported_reference():
    """Pins the restatement to the real thing: the unmodified reference's tensors for this case (pin_codec.npz)."""
    g = _pin("codec")
    sds = state_dicts(1)
    x, _ = case_inputs(dict(B=2, T=4500, xseed=21))
    with torch.no_grad():
        z2, q2, y2 = O.codec_forward(sds, x, n_c=2)
    for k, t in (("z", z2), ("outs", q2[0]), ("y", y2), ("timbre", q2[4]), ("z_p", q2[1][0]), ("z_c", q2[1][1]), ("z_r", q2[1][2])):
        _close(t, g[k], k)
    for k, t in zip(("codes_p", "codes_c", "codes_r"), q2[5]):
        assert np.array_equal(t.numpy(), g[k]), k
    _close(float(q2[2]), g["commitment"], "commitment")
    _close(float(q2[3]), g["codebook"], "codebook")


def test_fvq_rvq_and_alias_free_match_reference():
    g = _pin("rvq_act")
    sd = _pinned_params(g, 3)
    def wn(p):      # the projections are weight-normed (dim 0), as the reference module folds them
        return torch._weight_norm(sd[p + ".weight_v"], sd[p + ".weight_g"], 0)
    layers = [dict(in_w=wn(f"layers.{i}.in_proj"), in_b=sd[f"layers.{i}.in_proj.bias"],
                   out_w=wn(f"layers.{i}.out_proj"), out_b=sd[f"layers.{i}.out_proj.bias"],
                   codebook=sd[f"layers.{i}._codebook.weight"]) for i in range(4)]
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(2, 1024, 17, generator=gen)
    with torch.no_grad():
        b = O.fvq_residual_vq(layers, x)
    assert np.array_equal(b[1].numpy(), g["idx"])
    _close(b[0], g["q"], "q")
    _close(b[3], g["allq"], "allq")
    xx = torch.randn(2, 5, 50, generator=gen)
    _close(O.alias_free_act(xx, lambda u: u), g["act_y"], "alias-free")


def test_reflect_pad_short_branch():
    """encodec.py:96-113: length <= pad => zero-extend, reflect, truncate."""
    x = torch.arange(1, 4, dtype=torch.float32).reshape(1, 1, 3)
    y = O._pad1d_reflect(x, 5, 0)
    assert y.shape[-1] == 8
    assert y.flatten().tolist() == [0.0, 0.0, 0.0, 3.0, 2.0, 1.0, 2.0, 3.0]


# ---------------------------------------------------------------------------------------------------------------
# round 2: voice-conversion path (modules/redecoder.py), predictor heads (modules/quantize.py:29-125), dataset mel
# ---------------------------------------------------------------------------------------------------------------
from conftest import REDEC_CASES  # noqa: E402


def test_redecoder_case_table():
    from oracle import make_golden
    assert make_golden.REDEC_CASES == REDEC_CASES
    for name in REDEC_CASES:
        assert os.path.exists(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))


@pytest.mark.parametrize("name", list(REDEC_CASES))
def test_redecoder_oracle_matches_golden(name):
    from facodec_b200 import synth
    c = REDEC_CASES[name]
    g = load_golden(name)
    src = load_golden(c["src"])
    sds = synth.synth_redecoder_state_dicts(c["wseed"])
    cp, cc, timbre = (torch.from_numpy(src[k]) for k in ("codes_p", "codes_c", "timbre"))
    with torch.no_grad():
        z = O.redecoder_forward(sds["encoder"], cp, cc, timbre, use_p_code=c["use_p"], n_c=c["n_c"])
        y = O.decoder_forward(sds["decoder"], z, causal=False, lstm=0)
    _close(z, g["z"], "z")
    _close(y, g["y"], "y")


def test_redecoder_oracle_matches_imported_reference():
    """modules/redecoder.py:35-48 + the non-causal, LSTM-free Decoder of build_model(stage='redecoder') (pin_redecoder.npz)."""
    from facodec_b200 import synth
    pin = _pin("redecoder")
    sds = synth.synth_redecoder_state_dicts(2)
    g = torch.Generator().manual_seed(5)
    cp = torch.randint(0, 1024, (2, 1, 13), generator=g)
    cc = torch.randint(0, 1024, (2, 2, 13), generator=g)
    timbre = torch.randn(2, 1024, generator=g)
    for use_p, n_c in ((False, 1), (True, 2)):
        with torch.no_grad():
            z2 = O.redecoder_forward(sds["encoder"], cp, cc, timbre, use_p_code=use_p, n_c=n_c)
            y2 = O.decoder_forward(sds["decoder"], z2, causal=False, lstm=0)
        _close(z2, pin[f"z_{int(use_p)}{n_c}"], "z")
        _close(y2, pin[f"y_{int(use_p)}{n_c}"], "y")

def test_predictor_heads_and_snakebeta_match_imported_reference():
    """SnakeBeta (modules/quantize.py:29-88) inside Activation1d, the heads' ResidualUnit (:90-104) and CNNLSTM (:106-125)
    of the unmodified reference (pin_heads.npz)."""
    from facodec_b200 import synth
    pin = _pin("heads")
    g = torch.Generator().manual_seed(9)
    alpha = torch.randn(6, generator=g) * 0.3
    beta = torch.randn(6, generator=g) * 0.3
    x = torch.randn(2, 6, 40, generator=g)
    with torch.no_grad():
        _close(O.snake_beta(x, alpha, beta), pin["snakebeta"], "snakebeta")
        _close(O.alias_free_act(x, lambda u: O.snake_beta(u, alpha, beta)), pin["act"], "act")
    for j, (indim, outdim, heads, glob) in enumerate(((64, 10, 2, False), (32, 7, 1, True))):
        sd = synth.synth_cnnlstm(3, indim, outdim, heads)
        xx = torch.randn(2, indim, 33, generator=g)
        with torch.no_grad():
            b = O.cnnlstm_forward(sd, xx, heads, global_pred=glob)
        assert len(b) == heads
        for h, v in enumerate(b):
            _close(v, pin[f"cnnlstm{j}_head{h}"], f"cnnlstm{j} head {h}")

def test_dataset_mel_matches_imported_meldataset():
    """meldataset.py:37-47 preprocess (torchaudio MelSpectrogram with its default sample_rate = 16000) of the unmodified
    reference (pin_dataset_mel.npz: output, window, filterbank), against the restatement fed with the reference's window
    and filterbank and with synth's host-independent ones."""
    from facodec_b200 import synth
    pin = _pin("dataset_mel")
    w = synth.synth_waves(1, 5000, seed=3)[0, 0]
    ref = torch.from_numpy(pin["mel"])
    fb_ref, win_ref = torch.from_numpy(pin["fb"]), torch.from_numpy(pin["window"])
    with torch.no_grad():
        _close(O.dataset_mel(w, win_ref, fb_ref), pin["mel"], "mel")
        fb = synth.melscale_fbanks_htk(sample_rate=16000, f_max=8000.0)
        assert float((fb - fb_ref).abs().max()) <= 1e-5      # fp64-then-round vs torchaudio fp32 evaluation
        got = O.dataset_mel(w, synth.hann_window_periodic(1200), fb)
    assert tuple(ref.shape) == (1, 80, 5000 // 300 + 1)
    assert float((got - ref).abs().max()) <= 2e-5

def test_dac_code_file_matches_imported_dacfile(tmp_path):
    """dac/model/base.py:15-54: files written here are byte-identical to the reference class's (pin_dacfile.npz), and the
    reference's file loads here (codes, every metadata field)."""
    from facodec_b200 import codefile
    ref_bytes = _pin("dacfile")["bytes"].tobytes()
    g = torch.Generator().manual_seed(9)
    codes = [torch.randint(0, 1024, (2, n, 37), generator=g) for n in (1, 2, 3)]
    mine = codefile.from_forward(codes, original_length=37 * 300, input_db=torch.tensor([-23.5, -17.25]))
    pa = mine.save(tmp_path / "mine")
    assert pa.suffix == ".dac" and open(pa, "rb").read() == ref_bytes
    pb = tmp_path / "ref.dac"
    pb.write_bytes(ref_bytes)
    b = codefile.DACFile.load(pb)
    assert torch.equal(b.codes, codefile.pack_codes(codes))
    assert (b.chunk_length, b.original_length, b.channels, b.sample_rate, b.padding, b.dac_version) == (37, 11100, 1, 24000, True, "1.0.0")
    assert np.array_equal(np.asarray(b.input_db), np.array([-23.5, -17.25], np.float32))
    for u, v in zip(codefile.unpack_codes(b.codes, n_c=2), codes):
        assert torch.equal(u, v)

def _loss_signals(B=2, T=4800, seed=11):
    from facodec_b200 import synth
    return synth.synth_loss_pair(B, T, seed)


def test_reconstruction_loss_matches_imported_losses_py():
    """losses.py:65-89 of the unmodified reference (recon_loss.npz) against the restatement: the same scalar."""
    gold = np.load(os.path.join(ROOT, "tests", "golden", "recon_loss.npz"))
    x, G_x = _loss_signals(int(gold["B"]), int(gold["T"]), int(gold["seed"]))
    with torch.no_grad():
        got = O.reconstruction_loss(x, G_x)
    assert got.dim() == 0
    _close(np.float32(got), gold["loss"], "loss")


def test_reconstruction_loss_golden():
    """tests/golden/recon_loss.npz: loss + 13 terms the imported reference modules gave for the seeded pair (oracle/make_golden.py)."""
    import warnings
    warnings.simplefilter("ignore")
    gold = np.load(os.path.join(ROOT, "tests", "golden", "recon_loss.npz"))
    x, G_x = _loss_signals(int(gold["B"]), int(gold["T"]), int(gold["seed"]))
    with torch.no_grad():
        L, terms = O.reconstruction_loss(x, G_x, return_terms=True)
    assert abs(float(L) - float(gold["loss"])) <= 2e-6 * abs(float(gold["loss"]))
    assert np.allclose(terms.numpy(), gold["terms"], rtol=2e-6, atol=0)


FAP_FLAGS = dict(use_gr_content_f0=False, use_gr_prosody_phone=False, use_gr_residual_f0=True, use_gr_residual_phone=True,
                 use_gr_timbre_content=True, use_gr_timbre_prosody=False, use_gr_x_timbre=True, norm_f0=True)   # modules/commons.py:311-322 + config.yml


@pytest.mark.parametrize("timbre_norm", [True, False])
def test_fa_predictors_match_imported_reference(timbre_norm):
    """FApredictors (modules/quantize.py:456-619) of the unmodified reference with build_model's flags, both forward
    variants (pin_fa_predictors_*.npz: seeded parameters, sampled outputs): the restatement, output by output."""
    from oracle import make_golden
    pin = _pin(f"fa_predictors_{int(timbre_norm)}")
    sd = _pinned_params(pin, 4)
    g = torch.Generator().manual_seed(6)
    lat = [torch.randn(2, 32, 19, generator=g) for _ in range(3 if timbre_norm else 4)]
    with torch.no_grad():
        timbre = torch.randn(2, 32, generator=g) if timbre_norm else None
        got = O.fa_predictors_forward(sd, lat, timbre, timbre_norm=timbre_norm, **FAP_FLAGS)
    keys = {k for k in pin if k.startswith("out") and not k.startswith("outshape")}
    seen = set()
    for i, b in enumerate(got):
        for k, v in b.items():
            name = f"out{i}/{k}"
            if v is None:
                assert name not in pin, name
                continue
            assert tuple(v.shape) == tuple(pin[f"outshape{i}/{k}"]), name
            idx = torch.from_numpy(make_golden.sample_positions(v.numel()))
            # 1-wide nn.Linear heads (f0 / uv): torch's CPU F.linear takes another kernel for weights that do not require
            # grad (the oracle works on detached state_dict tensors, the module on Parameters): 1-2 ulp apart
            tol = 5e-7 if v.shape[-1] == 1 else ATOL
            a, r = v.reshape(-1)[idx].numpy(), pin[name]
            assert np.abs(a - r).max() <= tol * max(1.0, np.abs(r).max()), name
            seen.add(name)
    assert seen == keys


def test_slaney_mel_filterbank_against_torchaudio():
    """The restated librosa.filters.mel (Slaney scale + area norm; librosa itself is not installed) against torchaudio's
    independent Slaney implementation, for the geometries train.py:155-163 uses."""
    import torchaudio
    for w, nm in ((32, 5), (64, 10), (256, 40), (512, 80), (2048, 320), (2048, 150)):
        mine = O.librosa_mel_filters(24000, w, nm, 0.0, None)
        ref = torchaudio.functional.melscale_fbanks(w // 2 + 1, 0.0, 12000.0, nm, 24000, norm="slaney", mel_scale="slaney").T
        assert mine.shape == ref.shape == (nm, w // 2 + 1)
        assert float((mine - ref).abs().max()) <= 2e-6 * max(1.0, float(ref.abs().max())), (w, nm)


def test_dac_spectral_losses_restatement_properties():
    """dac/nn/loss.py MultiScaleSTFTLoss / MelSpectrogramLoss restatements (parity unpinned: audiotools absent): zero for
    identical signals, the magnitude path equals a direct torch.stft evaluation, train.py's mel configuration runs."""
    from facodec_b200 import synth
    x, y = synth.synth_loss_pair(2, 3000, seed=3)
    assert float(O.multiscale_stft_loss(x, x)) == 0.0
    assert float(O.mel_spectrogram_loss(x, x)) == 0.0
    st = torch.stft(x[:, 0], 512, hop_length=128, window=torch.hann_window(512), return_complex=True)
    sy = torch.stft(y[:, 0], 512, hop_length=128, window=torch.hann_window(512), return_complex=True)
    direct = (st.abs() - sy.abs()).abs().mean()
    got = O.multiscale_stft_loss(x, y, window_lengths=(512,), log_weight=0.0)
    assert abs(float(got) - float(direct)) <= 1e-6 * float(direct)
    L = O.mel_spectrogram_loss(x, y, 24000, n_mels=[5, 10, 20, 40, 80, 160, 320], window_lengths=[32, 64, 128, 256, 512, 1024, 2048],
                               mel_fmin=[0] * 7, mel_fmax=[None] * 7, pow=1.0, mag_weight=0.0)
    assert torch.isfinite(L) and float(L) > 0
