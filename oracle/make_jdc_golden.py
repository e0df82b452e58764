"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/pin_jdc.npz from the *unmodified* reference JDCNet.

    FACODEC_REFERENCE_ROOT=<reference tree> python -m oracle.make_jdc_golden

The fixture pins oracle/jdc_oracle.py (and through it the GPU JDCNet) to modules/JDC/model.py and train.py:
* the weights are facodec_b200.synth.synth_jdc(seed), regenerated from the stored seed (fixed-seed numpy draws, the same
  bits on every host); `weights_sha256` pins them, so a drift of the generator fails instead of silently moving the pin.
  Neither bst.t7 nor any reference source is stored.
* mel inputs of several T and the reference's eval-mode outputs (F0, GAN_feature, poolblock_out) on them, in fp32 as the
  reference computes them (model.py: x.float());
* modules/commons.py log_norm on those mels, and train.py:219-251's F0 targets as train.py computes them on the
  reference's F0 and on rows with no voiced frame, exactly one voiced frame and an inf F0.
"""
import hashlib
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from facodec_b200 import synth  # noqa: E402
from oracle import ref_import  # noqa: E402

SEED = 0
CASES = ((1, 1), (2, 5), (1, 37))          # (B, T) of the mel inputs


def weights_sha256(sd):
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(np.ascontiguousarray(v.detach().cpu().numpy()).tobytes())
    return h.hexdigest()


def mel_input(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 1, 80, T, generator=g) * 0.6 - 0.5).float()


def train_py_targets(F0_real):
    """train.py:219-251 (norm_f0) as written there; train.py has no importable function for it."""
    f0_targets, gt_glob_f0s = [], []
    for bib in range(len(F0_real)):
        voiced_indices = F0_real[bib] > 5.0
        f0_voiced = F0_real[bib][voiced_indices]
        if len(f0_voiced) != 0:
            log_f0 = f0_voiced.log2()
            mean_f0 = log_f0.mean()
            std_f0 = log_f0.std()
            normalized_f0 = (log_f0 - mean_f0) / std_f0
            normalized_sequence = torch.zeros_like(F0_real[bib])
            normalized_sequence[voiced_indices] = normalized_f0
            normalized_sequence[~voiced_indices] = -10
            gt_glob_f0s.append(mean_f0)
        else:
            normalized_sequence = torch.zeros_like(F0_real[bib]) - 10.0
            gt_glob_f0s.append(torch.tensor(0.0))
        f0_targets.append(normalized_sequence)
    f0_targets = torch.stack(f0_targets)
    f0_targets[torch.isnan(f0_targets)] = -10.0
    f0_targets[torch.isinf(f0_targets)] = -10.0
    return f0_targets, torch.stack(gt_glob_f0s)


def main():
    commons = ref_import.import_reference()
    spec = importlib.util.spec_from_file_location("_ref_jdc_model", os.path.join(ref_import.REFERENCE_ROOT, "modules", "JDC", "model.py"))
    model = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(model)
    sd = synth.synth_jdc(SEED)
    net = model.JDCNet(num_class=1, seq_len=192)
    net.load_state_dict(sd)
    net.eval()
    out = {"seed": np.int64(SEED), "weights_sha256": np.array(weights_sha256(sd)), "cases": np.array(CASES)}
    for i, (B, T) in enumerate(CASES):
        x = mel_input(B, T, 100 + i)
        with torch.no_grad():
            f0, gan, pool = net(x)
            ln = commons.log_norm(x).squeeze(1)
        out[f"mel_{i}"] = x.numpy()
        out[f"f0_{i}"] = f0.numpy()
        out[f"gan_{i}"] = gan.numpy()
        out[f"pool_{i}"] = pool.numpy()
        out[f"log_norm_{i}"] = ln.numpy()
    # targets: the reference F0 of the T = 37 case, plus rows with no / one voiced frame and an inf F0
    f0 = torch.from_numpy(out["f0_2"]).clone()
    T = f0.shape[1]
    extra = torch.zeros(3, T)
    extra[1, 11] = 220.0
    extra[2] = f0[0] + 1.0
    extra[2, 3] = float("inf")
    f0_in = torch.cat([f0, extra])
    tg, glob = train_py_targets(f0_in)
    out["targets_f0"] = f0_in.numpy()
    out["targets"] = tg.numpy()
    out["targets_glob"] = glob.numpy()
    path = os.path.join(ROOT, "tests", "golden", "pin_jdc.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
