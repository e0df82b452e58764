"""Host checks of the JDCNet surface: state-dict keys, the fp64 restatement's targets against train.py's loop, and -- where
the reference tree is present (FACODEC_REFERENCE_ROOT) -- the restatement against the unmodified reference JDCNet and the
real bst.t7 key set."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import facodec_b200 as fb
from facodec_b200 import synth
from oracle import jdc_oracle as O

REF = os.environ.get("FACODEC_REFERENCE_ROOT", "")
PIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pin_jdc.npz")


def _ref_jdc():
    path = os.path.join(REF, "modules", "JDC", "model.py")
    if not REF or not os.path.exists(path):
        pytest.skip("reference tree not present (FACODEC_REFERENCE_ROOT)")
    spec = importlib.util.spec_from_file_location("_ref_jdc_model", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.JDCNet


def test_synth_weights_match_the_state_dict():
    sd = synth.synth_jdc(0)
    m = fb.JDCNet()
    assert list(sd.keys()) == list(m.state_dict().keys())
    m.load_state_dict(sd)
    assert torch.equal(m.state_dict()["classifier.bias"], sd["classifier.bias"])
    assert (sd["res_block2.conv.1.running_var"] != 1).all() and (sd["pool_block.0.running_mean"] != 0).all()


def test_train_mode_and_num_class():
    with pytest.raises(ValueError):
        fb.JDCNet(num_class=722)
    m = fb.JDCNet()
    with pytest.raises(NotImplementedError):
        m.train()(torch.zeros(1, 1, 80, 4))


def _train_py_targets(F0):
    """train.py:223-251 as written there (fp64 inputs)."""
    out, glob = [], []
    for bib in range(len(F0)):
        voiced = F0[bib] > 5.0
        fv = F0[bib][voiced]
        if len(fv) != 0:
            lf = fv.log2()
            mean, std = lf.mean(), lf.std()
            seq = torch.zeros_like(F0[bib])
            seq[voiced] = (lf - mean) / std
            seq[~voiced] = -10
            glob.append(mean)
        else:
            seq = torch.zeros_like(F0[bib]) - 10.0
            glob.append(torch.tensor(0.0, dtype=F0.dtype))
        out.append(seq)
    out = torch.stack(out)
    out[torch.isnan(out)] = -10.0
    out[torch.isinf(out)] = -10.0
    return out, torch.stack(glob)


def test_oracle_targets_restate_train_py():
    g = torch.Generator().manual_seed(3)
    f0 = torch.rand(5, 64, generator=g, dtype=torch.float64) * 300
    f0[f0 < 60] = 0
    f0[1] = 0
    f0[2] = 0
    f0[2, 9] = 180.0
    f0[3, 4] = float("inf")
    a, ga = O.f0_targets(f0)
    b, gb = _train_py_targets(f0)
    assert torch.equal(a, b)
    assert torch.equal(ga.isinf(), gb.isinf()) and torch.equal(ga[~ga.isinf()], gb[~gb.isinf()])


def test_oracle_log_norm_restates_commons():
    x = torch.randn(2, 1, 80, 30, dtype=torch.float64)
    ref = torch.log(torch.exp(x * 4 + -4).norm(dim=2)).squeeze(1)
    assert torch.allclose(O.log_norm(x[:, 0]), ref, rtol=1e-14, atol=0)


def test_oracle_against_reference_jdcnet():
    JDC = _ref_jdc()
    sd = synth.synth_jdc(1)
    ref = JDC(num_class=1, seq_len=192)
    ref.load_state_dict(sd)
    ref.eval()
    x = torch.randn(2, 1, 80, 37, generator=torch.Generator().manual_seed(5)) * 0.6 - 0.5
    with torch.no_grad():
        f0, gan, pool = ref(x)            # the reference computes in fp32 (x.float())
    for dt, tol in ((torch.float32, 2e-5), (torch.float64, 1e-4)):
        o = O.jdc_forward(sd, x, dtype=dt)
        for a, r in zip(o[:3], (f0, gan, pool)):
            assert (a.double() - r.double()).abs().max() <= tol * max(1.0, r.abs().max().item())


def test_bst_t7_keys_load():
    path = os.path.join(REF, "modules", "JDC", "bst.t7")
    if not REF or not os.path.exists(path):
        pytest.skip("reference tree not present (FACODEC_REFERENCE_ROOT)")
    m = fb.load_F0_models(path)
    assert not m.training
    assert set(torch.load(path, map_location="cpu")["net"].keys()) == set(m.state_dict().keys())


def test_oracle_against_pinned_reference_outputs():
    """pin_jdc.npz (oracle/make_jdc_golden.py): the unmodified reference JDCNet's eval-mode outputs on synth_jdc weights,
    modules/commons.py log_norm and train.py's F0 targets."""
    from oracle.make_jdc_golden import weights_sha256
    pin = np.load(PIN)
    sd = synth.synth_jdc(int(pin["seed"]))
    assert weights_sha256(sd) == str(pin["weights_sha256"]), "synth_jdc no longer draws the pinned weights"
    for i in range(len(pin["cases"])):
        x = torch.from_numpy(pin[f"mel_{i}"])
        f0, gan, pool, _ = O.jdc_forward(sd, x)
        for name, got in (("f0", f0), ("gan", gan), ("pool", pool)):
            ref = torch.from_numpy(pin[f"{name}_{i}"]).double()
            # the reference runs in fp32: its own rounding, ~1e-7 relative, is what separates it from the fp64 restatement
            assert (got - ref).abs().max() <= 2e-5 * max(1.0, ref.abs().max().item()), (name, i)
        ln = torch.from_numpy(pin[f"log_norm_{i}"]).double()
        assert (O.log_norm(x[:, 0]) - ln).abs().max() <= 1e-5 * max(1.0, ln.abs().max().item())
    tg, glob = O.f0_targets(torch.from_numpy(pin["targets_f0"]))
    rtg, rglob = torch.from_numpy(pin["targets"]).double(), torch.from_numpy(pin["targets_glob"]).double()
    assert torch.equal(tg == -10.0, rtg == -10.0)
    assert (tg - rtg).abs().max() <= 1e-4
    fin = torch.isfinite(rglob)
    assert torch.equal(fin, torch.isfinite(glob)) and (glob[fin] - rglob[fin]).abs().max() <= 1e-6
