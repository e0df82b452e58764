"""TEST INFRASTRUCTURE ONLY -- decoding from codes: the CPU restatement and the generator of its reference pin.

The reference has no single call that turns codes back into the decoder's input.  Its FAquantizer.decode
(modules/quantize.py:245-254) is written for the timbre-quantizer variant: it splits the codes [1, 1, 2] and calls
self.timbre_quantizer, which does not exist when timbre_norm = True (the shipped config), so it raises.  The semantics
restated here are the composition of reference pieces:

    z_p = prosody_quantizer.from_codes(codes_p)[0]       dac/nn/quantize.py:200-220
    z_c = content_quantizer.from_codes(codes_c)[0]       1 or 2 rows
    z_r = residual_quantizer.from_codes(codes_r)[0]      1..3 rows; 0 rows = left out, as res_mask = 0 does (:419-437)
    outs = LayerNorm((z_p + z_c) + z_r) * gamma + beta   gamma | beta = timbre_linear(timbre), modules/quantize.py:444-449

Only tests/ import quantizer_from_codes.  ``python -m oracle.from_codes`` writes tests/golden/pin_from_codes.npz from the
imported, unmodified reference (needs the reference tree, see oracle/ref_import.py) and touches no other fixture.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.facodec_oracle import _wn_weight  # noqa: E402

GOLDEN_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")


def rvq_from_codes(sd, prefix, codes, dtype=torch.float32):
    """ResidualVectorQuantize.from_codes, dac/nn/quantize.py:200-220: z_q = 0.0 + sum_i out_proj_i(codebook_i[codes_i])
    (VectorQuantize.decode_code = F.embedding on the raw codebook, :72-76)."""
    z_q = 0.0
    for i in range(codes.shape[1]):
        pre = f"{prefix}.quantizers.{i}"
        z_p_i = F.embedding(codes[:, i, :], sd[pre + ".codebook.weight"].to(dtype)).transpose(1, 2)
        w_out = _wn_weight({k: v.to(dtype) for k, v in sd.items() if k.startswith(pre + ".out_proj")}, pre + ".out_proj")
        z_q = z_q + F.conv1d(z_p_i, w_out, sd[pre + ".out_proj.bias"].to(dtype))
    return z_q


def quantizer_from_codes(sd, codes_p, codes_c, codes_r, timbre, dtype=torch.float32):
    """FAquantizer decoding from codes (module docstring) on the quantizer's state_dict.  codes_r may be None or have 0
    rows: z_r is then zeros and outs = z_p + z_c.  dtype float64 gives an fp64 reference for the kernel tests.
    Returns (outs [B,1024,T], [z_p, z_c, z_r])."""
    with torch.no_grad():
        z_p = rvq_from_codes(sd, "prosody_quantizer", codes_p, dtype)
        z_c = rvq_from_codes(sd, "content_quantizer", codes_c, dtype)
        outs = z_p + z_c
        if codes_r is not None and codes_r.shape[1] > 0:
            z_r = rvq_from_codes(sd, "residual_quantizer", codes_r, dtype)
            outs = outs + z_r
        else:
            z_r = torch.zeros_like(z_p)
        style = F.linear(timbre.to(dtype), sd["timbre_linear.weight"].to(dtype), sd["timbre_linear.bias"].to(dtype)).unsqueeze(2)
        gamma, beta = style.chunk(2, 1)
        o = F.layer_norm(outs.transpose(1, 2), (outs.shape[1],), None, None, 1e-5).transpose(1, 2)
        return o * gamma + beta, [z_p, z_c, z_r]


# (content rows, residual rows) of the seeded random pin cases; utterances and frames per random case
RANDOM_ROWS = ((1, 3), (2, 1), (2, 0))
RANDOM_B, RANDOM_T = 2, 6


def random_case(n_c, n_r):
    """Seeded random codes of one pin case, with indices 0 and 1023 present in every code tensor that has rows, and a
    seeded random timbre."""
    g = torch.Generator().manual_seed(100 + 10 * n_c + n_r)
    codes = []
    for rows in (1, n_c, n_r):
        c = torch.randint(0, 1024, (RANDOM_B, rows, RANDOM_T), generator=g)
        if rows:
            c[0, 0, 0], c[-1, -1, -1] = 0, 1023
        codes.append(c)
    return codes, torch.randn(RANDOM_B, 1024, generator=g)


def main():
    """tests/golden/pin_from_codes.npz with the imported reference (synthetic checkpoint 1, as pin_codec):
    ResidualVectorQuantize.from_codes of the FAquantizer's three quantizers, timbre_linear / timbre_norm as forward_v2
    applies them, then the decoder.  Cases: the codes and timbre of the pin_codec forward, and random codes at RANDOM_ROWS.
    With no residual rows the reference cannot call from_codes (it ends in torch.cat of an empty list); outs is then
    z_p + z_c through the same AdaLN."""
    import warnings
    warnings.simplefilter("ignore")
    from facodec_b200 import synth
    from oracle import ref_import
    ref_import.import_reference()
    model = ref_import.build_reference_model(0)
    sds = synth.synth_state_dicts(1)
    for k in ("encoder", "quantizer", "decoder"):
        model[k].load_state_dict(sds[k])
    qz = model.quantizer
    x = synth.synth_waves(2, 4500, seed=21)          # the pin_codec input
    with torch.no_grad():
        q = qz(model.encoder(x), x, n_c=2, return_codes=True)
    cases = {"codec": (list(q[5]), q[4])}
    for n_c, n_r in RANDOM_ROWS:
        cases[f"c{n_c}r{n_r}"] = random_case(n_c, n_r)
    d = {}
    for name, ((cp, cc, cr), timbre) in cases.items():
        with torch.no_grad():
            z_p = qz.prosody_quantizer.from_codes(cp)[0]
            z_c = qz.content_quantizer.from_codes(cc)[0]
            outs = z_p + z_c
            z_r = torch.zeros_like(z_p)
            if cr.shape[1]:
                z_r = qz.residual_quantizer.from_codes(cr)[0]
                outs = outs + z_r
            gamma, beta = qz.timbre_linear(timbre).unsqueeze(2).chunk(2, 1)
            outs = qz.timbre_norm(outs.transpose(1, 2)).transpose(1, 2) * gamma + beta
            y = model.decoder(outs)
        d.update({f"{name}/{k}": v for k, v in dict(codes_p=cp, codes_c=cc, codes_r=cr, timbre=timbre, outs=outs, z_p=z_p,
                                                     z_c=z_c, z_r=z_r, y=y).items()})
    path = os.path.join(GOLDEN_DIR, "pin_from_codes.npz")
    np.savez_compressed(path, **{k: v.detach().numpy() for k, v in d.items()})
    print("from_codes", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
