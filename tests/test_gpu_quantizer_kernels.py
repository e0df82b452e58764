"""GPU: the quantizer-side kernels (quant.cu, frontend.cu) against plain float64 references at chosen inputs.

* fa_quantize_kernel (the six fused VectorQuantizes + the AdaLN) through fac_debug_fa_quantize: random frames with the
  decidable-frame rule below, and exact ties placed on one lane, on adjacent lanes and across the whole index range.
* rvq_kernel through fb.ResidualVQ: the same ties, frame counts around its 16-frame CTA, nq = 1 and nq = 8.
* attention_kernel / attention_stream_kernel through fac_debug_attention: masks, ragged T, both kernels, the switch
  between them at T = 2430 / 2431.
* The masked timbre path (valid_len row masks, the second GLU's mask, mean_pool over valid frames) end to end.
* The mel front-end ("mel80" tap): the frames gather + tensor-core DFT and the fp32 strided-conv DFT.

Rounding bounds use u = 2^-24 (fp32 unit roundoff) and gamma_n = n u / (1 - n u) (Higham, Accuracy and Stability of
Numerical Algorithms, 2nd ed., section 3.1): a sum in which each term passes through at most n roundings is within
gamma_n * sum |terms| of the exact sum.

Decidable frames: a VQ decision is decidable when the fp64 reference's top-1 / top-2 distance gap exceeds delta, the
largest amount the kernel's fp32 distances can move that gap.  delta is computed per decision from the frame itself:
  - z_e = in_w r + b: each lane chains 32 FMAs, then 5 shuffle adds and the bias, so |dz_e_k| <= gamma_38 sum_i |w_ki r_i|
    + sum_i |w_ki| eps_r_i + u |z_e_k|, where eps_r (per channel) bounds the error of the residual r the stage receives
    (0 for the first stage; it grows by the fp32 out-projection error of each earlier stage, see _Chain);
  - F.normalize (8-term norm, sqrt, divide): ||d enc|| <= 2 ||dz_e|| / ||z_e|| + 8u;
  - dist_j = |enc|^2 - 2 enc . cbn_j + |cbn_j|^2: |enc|^2 is the same value for every code and cancels in the gap; the
    8-term dot moves by <= ||d enc|| + gamma_8 + 8u (cbn_j rounded to fp32 on the host), the packed |cbn_j|^2 by
    <= 32u, the two fp32 roundings of the sum (values <= 4) by <= 8u;  so each distance moves by
    <= 2 ||d enc|| + 2 gamma_8 + 56u and the gap by twice that:
  delta = 4 ||d enc|| + 4 gamma_8 + 112u, rounded up to 4 ||d enc|| + 4 gamma_8 + 128u.
Frames whose six (or nq) decisions are all decidable must get the reference's codes exactly.  Exact ties (margin 0)
are tested separately: the kernel must return the lower index, as torch's first-maximum rule does.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def gamma(n):
    return n * U / (1 - n * U)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


_MODEL = {}


def _model(seed):
    import facodec_b200 as fb
    from conftest import state_dicts
    if seed not in _MODEL:
        _MODEL.clear()
        m = fb.build_model()
        sds = state_dicts(seed)
        for k in ("encoder", "quantizer", "decoder"):
            m[k].load_state_dict(sds[k])
            m[k].eval()
        _MODEL[seed] = m
    return _MODEL[seed]


def _engine():
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    return e


# ---------------------------------------------------------------------------------------------------------------------
# fp64 residual-VQ chain with per-decision margins and error bounds
# ---------------------------------------------------------------------------------------------------------------------
class _Chain:
    """One ResidualVectorQuantize (dac/nn/quantize.py:127-198, eval) in float64 on frames [N][1024], with, per stage:
    codes, the top-1/top-2 gap, the decidability bound delta (module docstring), and elementwise bounds on the error of
    the fp32 kernel's stage outputs and residual given the same codes."""

    def __init__(self, vqs, x, eps_in=None):
        """vqs: list of dicts in_w [8][1024], in_b [8], out_w [1024][8], out_b [1024], codebook [1024][8] (fp32);
        x: [N][1024] fp64 input; eps_in: [N][1024] bound on the input's error (None = exact)."""
        r = x.clone()
        eps_r = torch.zeros_like(x) if eps_in is None else eps_in.clone()
        self.codes, self.margin, self.delta, self.se, self.se_bound, self.outs = [], [], [], [], [], []
        self.out_err = torch.zeros_like(x)                       # bound on |sum of stage outputs - reference|
        qsum = torch.zeros_like(x)
        for v in vqs:
            w = v["in_w"].double()
            cb = v["codebook"].double()
            wo = v["out_w"].double()
            ze = r @ w.t() + v["in_b"].double()
            dze = gamma(38) * (r.abs() @ w.abs().t()) + eps_r @ w.abs().t() + U * ze.abs()
            denc = 2 * dze.norm(dim=1) / ze.norm(dim=1).clamp_min(1e-12) + 8 * U
            enc = F.normalize(ze)
            cbn = F.normalize(cb)
            dist = enc.pow(2).sum(1, keepdim=True) - 2 * enc @ cbn.t() + cbn.pow(2).sum(1)[None, :]
            top2 = torch.topk(-dist, 2, dim=1)
            idx = (-dist).max(1)[1]
            zq = cb[idx]
            out = zq @ wo.t() + v["out_b"].double()
            # fp32 stage output given the same code: zq = ze + (cb - ze) rounds twice (<= 2u (|cb| + |ze|) per k), the
            # 8-term out-projection + bias chains 9 FMAs (gamma_9); the residual update rounds once more (u |r'|)
            e_out = gamma(11) * ((cb[idx].abs() + ze.abs()) @ wo.abs().t() + v["out_b"].double().abs())
            r = r - out
            qsum = qsum + out
            eps_r = eps_r + e_out + U * r.abs()
            self.out_err = self.out_err + e_out + U * qsum.abs()
            d = ze - zq
            se = d.pow(2).sum(1)
            # se = sum_k (z_e - z_q)^2 over 8 fp32 FMAs
            self.se_bound.append(2 * (d.abs() * dze).sum(1) + dze.pow(2).sum(1) + gamma(9) * se)
            self.se.append(se)
            self.codes.append(idx)
            self.margin.append(top2.values[:, 0] - top2.values[:, 1])
            self.delta.append(4 * denc + 4 * gamma(8) + 128 * U)
            self.outs.append(out)
        self.qsum = qsum
        self.residual = r
        self.eps_r = eps_r                                       # bound on |kernel residual - reference|

    def decidable(self):
        ok = torch.ones_like(self.codes[0], dtype=torch.bool)
        for m, d in zip(self.margin, self.delta):
            ok &= m > d
        return ok


def _quantizer_vqs(sd):
    from oracle import facodec_oracle as O
    out = []
    for pre in ["prosody_quantizer.quantizers.0", "content_quantizer.quantizers.0", "content_quantizer.quantizers.1",
                "residual_quantizer.quantizers.0", "residual_quantizer.quantizers.1", "residual_quantizer.quantizers.2"]:
        out.append(dict(in_w=O._wn_weight(sd, pre + ".in_proj").reshape(8, 1024).float().contiguous(),
                        in_b=sd[pre + ".in_proj.bias"].float().contiguous(),
                        out_w=O._wn_weight(sd, pre + ".out_proj").reshape(1024, 8).float().contiguous(),
                        out_b=sd[pre + ".out_proj.bias"].float().contiguous(),
                        codebook=sd[pre + ".codebook.weight"].float().contiguous()))
    return out


def _fa_reference(vqs, f0, z, gb, n_c):
    """FAquantizer.forward_v2's VQ half (modules/quantize.py:421-454) in fp64 on frames [N][1024]; gb [N][2048]."""
    x = z.double()
    p = _Chain(vqs[0:1], f0.double())
    c = _Chain(vqs[1:1 + n_c], x)
    rin = x - p.qsum - c.qsum
    r = _Chain(vqs[3:6], rin, eps_in=p.out_err + c.out_err + 2 * U * rin.abs())
    s = p.qsum + c.qsum + r.qsum
    eps_s = p.out_err + c.out_err + r.out_err + 2 * U * s.abs()
    mu = s.mean(1, keepdim=True)
    var = (s - mu).pow(2).mean(1, keepdim=True)
    rstd = (var + 1e-5).rsqrt()
    xn = (s - mu) * rstd
    g, b = gb[:, :1024].double(), gb[:, 1024:].double()
    outs = xn * g + b
    # LayerNorm in fp32 (per-lane chains of 32 + 5 shuffle adds for the mean and the variance):
    #   |d mean| <= mean(eps_s) + gamma_37 mean|s|;  |d var| <= 2 mean((eps_s + |d mean|) |s - mu|) + gamma_38 var;
    #   rsqrt: |d rstd| / rstd <= |d var| / (2 (var + 1e-5)) + 2u;
    #   |d xn| <= rstd (eps_s + |d mean|) + |xn| (|d rstd| / rstd + 2u);  |d outs| <= |g| |d xn| + 2u (|g xn| + |b|)
    dmu = eps_s.mean(1, keepdim=True) + gamma(37) * s.abs().mean(1, keepdim=True)
    dvar = 2 * ((eps_s + dmu) * (s - mu).abs()).mean(1, keepdim=True) + gamma(38) * var
    rrel = dvar / (2 * (var + 1e-5)) + 2 * U
    dxn = rstd * (eps_s + dmu) + xn.abs() * (rrel + 2 * U)
    douts = g.abs() * dxn + 2 * U * ((g * xn).abs() + b.abs())
    return p, c, r, outs, douts


def _run_fa_quantize(vqs, f0, z, gb, n_c, B, Tq, Tz, Tf0):
    e = _engine()
    dev = "cuda"
    keep = []
    rows = (ctypes.c_void_p * 5) * 6
    arr = rows()
    for i, v in enumerate(vqs):
        for j, k in enumerate(("in_w", "in_b", "out_w", "out_b", "codebook")):
            t = v[k].contiguous()
            keep.append(t)
            arr[i][j] = t.data_ptr()
    f0d, zd, gbd = f0.to(dev).contiguous(), z.to(dev).contiguous(), gb.to(dev).contiguous()
    nan = float("nan")
    outs = torch.full((B, Tq, 1024), nan, device=dev)
    zp, zc, zr = (torch.full((B, Tq, 1024), nan, device=dev) for _ in range(3))
    cp = torch.full((B, 1, Tq), -1, dtype=torch.int64, device=dev)
    cc = torch.full((B, n_c, Tq), -1, dtype=torch.int64, device=dev)
    cr = torch.full((B, 3, Tq), -1, dtype=torch.int64, device=dev)
    sqerr = torch.full((6, B * Tq), nan, device=dev)
    losses = torch.full((2,), nan, device=dev)
    rc = e.L.fac_debug_fa_quantize(e.handle, _p(f0d), _p(zd), ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p)), _p(gbd),
                                   n_c, B, Tq, Tz, Tf0, _p(outs), _p(zp), _p(zc), _p(zr), _p(cp), _p(cc), _p(cr), _p(sqerr),
                                   _p(losses), None)
    assert rc == 0, e.L.fac_last_error(e.handle)
    # the product passes NULL for the parts when the caller does not want them: same codes and outs
    outs2 = torch.full_like(outs, nan)
    cp2, cc2, cr2 = torch.full_like(cp, -1), torch.full_like(cc, -1), torch.full_like(cr, -1)
    rc = e.L.fac_debug_fa_quantize(e.handle, _p(f0d), _p(zd), ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p)), _p(gbd),
                                   n_c, B, Tq, Tz, Tf0, _p(outs2), None, None, None, _p(cp2), _p(cc2), _p(cr2),
                                   _p(sqerr), _p(losses), None)
    assert rc == 0, e.L.fac_last_error(e.handle)
    assert torch.equal(outs, outs2) and torch.equal(cp, cp2) and torch.equal(cc, cc2) and torch.equal(cr, cr2)
    return [t.cpu() for t in (outs, zp, zc, zr, cp, cc, cr, sqerr, losses)]


def _frames(t, B, Tq):
    """[B][T'][1024] -> the [B*Tq][1024] frames the kernel reads (t < Tq of every utterance)."""
    return t[:, :Tq].reshape(B * Tq, -1)


@pytest.mark.parametrize("n_c,B,Tq", [(1, 3, 7), (2, 3, 7), (2, 2, 37), (1, 3, 101), (2, 3, 101)])
def test_fa_quantize_random_frames(n_c, B, Tq, built_lib):
    from conftest import state_dicts
    vqs = _quantizer_vqs(state_dicts(0)["quantizer"])
    g = torch.Generator().manual_seed(1000 * n_c + 10 * B + Tq)
    Tz, Tf0 = Tq + 5, Tq + 3          # the kernel steps through z and f0 with their own strides
    f0 = torch.randn(B, Tf0, 1024, generator=g)
    z = torch.randn(B, Tz, 1024, generator=g)
    gb = torch.cat([1 + 0.2 * torch.randn(B, 1024, generator=g), 0.2 * torch.randn(B, 1024, generator=g)], 1)
    outs, zp, zc, zr, cp, cc, cr, sqerr, losses = _run_fa_quantize(vqs, f0, z, gb, n_c, B, Tq, Tz, Tf0)
    N = B * Tq
    p, c, r, outs_ref, douts = _fa_reference(vqs, _frames(f0, B, Tq), _frames(z, B, Tq),
                                             gb.repeat_interleave(Tq, 0), n_c)
    ok = p.decidable() & c.decidable() & r.decidable()
    n_bad = int((~ok).sum())
    print(f"FAQ n_c={n_c} frames={N} undecidable={n_bad} "
          f"delta median={torch.cat([torch.stack(ch.delta) for ch in (p, c, r)], 0).median().item():.2e}")
    # a decision is undecidable with probability ~ delta / (typical top-2 gap): delta ~ 4e-4 (first stages) to 1.3e-3
    # (residual stages, whose input carries the earlier stages' error) against a median gap ~ 0.05 leaves ~7 % of frames
    # with at least one undecidable decision among six
    assert n_bad <= max(3, N // 8), f"{n_bad} of {N} frames undecidable"
    assert ok.any()
    kcodes = [cp.reshape(B, 1, Tq), cc.reshape(B, n_c, Tq), cr.reshape(B, 3, Tq)]
    for name, ch, kc in zip(("prosody", "content", "residual"), (p, c, r), kcodes):
        for q, ref in enumerate(ch.codes):
            got = kc[:, q, :].reshape(N)
            assert torch.equal(got[ok], ref[ok]), f"{name}[{q}]: {int((got[ok] != ref[ok]).sum())} decidable codes differ"
    # parts: fp32 stage outputs vs fp64, per frame (bounds from _Chain)
    for name, ch, t in (("zp", p, zp), ("zc", c, zc), ("zr", r, zr)):
        err = (t.reshape(N, 1024).double() - ch.qsum).abs()
        assert (err[ok] <= ch.out_err[ok]).all(), f"{name}: max err/bound {(err[ok] / ch.out_err[ok]).max():.2f}"
    err = (outs.reshape(N, 1024).double() - outs_ref).abs()
    assert (err[ok] <= douts[ok]).all(), f"outs: max err {err[ok].max():.3e}"
    # sqerr rows: prosody, content 0, content 1 (exactly 0 when n_c = 1), residual 0..2
    rows = [p.se[0], c.se[0], c.se[1] if n_c == 2 else None] + r.se
    bounds = [p.se_bound[0], c.se_bound[0], c.se_bound[1] if n_c == 2 else None] + r.se_bound
    for q in range(6):
        got = sqerr[q].double()
        if rows[q] is None:
            assert torch.equal(sqerr[q], torch.zeros(N)), "sqerr row 2 must be exactly 0 when n_c = 1"
            continue
        assert ((got - rows[q]).abs()[ok] <= bounds[q][ok]).all(), f"sqerr row {q}"
    # losses: commitment = codebook = sum_q mean_b(sum_t sqerr / (8 Tq)), accumulated in fp64 then rounded to fp32
    total = float(sqerr.double().sum() / (8.0 * Tq * B))
    assert losses[0].item() == losses[1].item()
    assert abs(losses[0].item() - total) <= 2 * U * abs(total)
    if n_bad == 0:
        ref_total = float(sum(s.sum() for s in rows if s is not None) / (8.0 * Tq * B))
        bound = float(sum(b.sum() for b in bounds if b is not None) / (8.0 * Tq * B)) + 2 * U * abs(ref_total)
        assert abs(losses[0].item() - ref_total) <= bound


# codebook rows duplicated so that two codes are equal in the kernel's own arithmetic (identical packed rows give the
# identical fp32 distance): the same lane (j, j + 32 k), adjacent lanes (j, j + 1), including lane 31 -> lane 0 of the
# next sweep (63, 64), and the ends of the range (0, 1023)
TIE_PAIRS = [(5, 5 + 32 * 7), (100, 100 + 32 * 20), (40, 41), (63, 64), (0, 1023)]


def _with_ties(v):
    cb = v["codebook"].clone()
    for a, b in TIE_PAIRS:
        cb[b] = cb[a]
    return dict(v, codebook=cb.contiguous())


def _frame_on_code(v, j, scale):
    """A frame r with in_w r + in_b = scale * codebook[j] (least squares: in_w is 8 x 1024 of full row rank)."""
    w = v["in_w"].double()
    t = scale * v["codebook"][j].double() - v["in_b"].double()
    return torch.linalg.lstsq(w, t[:, None]).solution[:, 0]


@pytest.mark.parametrize("n_c", [1, 2])
def test_fa_quantize_exact_ties_pick_lower_index(n_c, built_lib):
    from conftest import state_dicts
    vqs = [_with_ties(v) for v in _quantizer_vqs(state_dicts(1)["quantizer"])]
    g = torch.Generator().manual_seed(77 + n_c)
    B, Tq = 2, 11
    Tz, Tf0 = Tq + 1, Tq + 2
    f0 = torch.randn(B, Tf0, 1024, generator=g)
    z = torch.randn(B, Tz, 1024, generator=g)
    gb = torch.cat([torch.ones(B, 1024), torch.zeros(B, 1024)], 1)
    # prosody ties on frames (b, t) = slots 0..9, content-0 ties on the other pair member's slots; both members of each
    # pair appear as the target (the kernel sees the same distance either way)
    slots = [(0, 0), (0, 3), (0, 5), (0, 10), (1, 0), (1, 4), (1, 9), (1, 10), (0, 7), (1, 6)]
    targets = [j for pair in TIE_PAIRS for j in pair]
    for (b, t), j in zip(slots, targets):
        f0[b, t] = _frame_on_code(vqs[0], j, 1.5).float()
        z[b, t] = _frame_on_code(vqs[1], targets[(targets.index(j) + 1) % len(targets)], 0.7).float()
    outs, zp, zc, zr, cp, cc, cr, sqerr, losses = _run_fa_quantize(vqs, f0, z, gb, n_c, B, Tq, Tz, Tf0)
    p = _Chain(vqs[0:1], _frames(f0, B, Tq).double())
    c = _Chain(vqs[1:1 + n_c], _frames(z, B, Tq).double())
    lower = {a: a for a, _ in TIE_PAIRS}
    lower.update({b_: a for a, b_ in TIE_PAIRS})
    for (b, t), j in zip(slots, targets):
        jc = targets[(targets.index(j) + 1) % len(targets)]
        n = b * Tq + t
        assert int(p.codes[0][n]) == lower[j] and int(c.codes[0][n]) == lower[jc]   # torch: first maximum
        assert int(cp[b, 0, t]) == lower[j], f"prosody tie {j}: kernel chose {int(cp[b, 0, t])}"
        assert int(cc[b, 0, t]) == lower[jc], f"content tie {jc}: kernel chose {int(cc[b, 0, t])}"


# ---------------------------------------------------------------------------------------------------------------------
# rvq_kernel through the public ResidualVQ
# ---------------------------------------------------------------------------------------------------------------------
def _rvq_layers(rvq):
    n = rvq.num_quantizers
    return [dict(in_w=rvq._folded(i, "in_proj"), in_b=rvq._p[f"layers/{i}/in_proj/bias"].detach().clone(),
                 out_w=rvq._folded(i, "out_proj"), out_b=rvq._p[f"layers/{i}/out_proj/bias"].detach().clone(),
                 codebook=rvq._p[f"layers/{i}/_codebook/weight"].detach().clone()) for i in range(n)]


@pytest.mark.parametrize("nq", [1, 8])
@pytest.mark.parametrize("B,T", [(1, 1), (1, 15), (1, 17), (3, 11), (1, 16 * 5 + 1)])
def test_rvq_ties_and_tails(B, T, nq, built_lib):
    """B*T = 1, 15, 17, 33 = 16*2 + 1, 81 = 16*5 + 1 frames: the CTA holds 16 frames and repeats the last one in its tail."""
    import facodec_b200 as fb
    from oracle import facodec_oracle as O
    rvq = fb.ResidualVQ(num_quantizers=nq, codebook_size=10, dim=1024, codebook_dim=8, seed=3).eval()
    sd = rvq.state_dict()
    for i in range(nq):
        k = f"layers.{i}._codebook.weight"
        sd[k] = _with_ties(dict(codebook=sd[k]))["codebook"]
    rvq.load_state_dict(sd)
    layers = _rvq_layers(rvq)
    N = B * T
    g = torch.Generator().manual_seed(N * 10 + nq)
    x = torch.randn(N, 1024, generator=g, dtype=torch.float64)
    # stage-0 ties on the last frame (the tail's repeated frame) and spread over the rest; cross-lane pairs first, so
    # that even one frame meets the shuffle reduction's tie rule
    targets = [1023, 0, 41, 40, 64, 63, 229, 5, 740, 100]
    tie_frames = sorted({N - 1} | set(range(0, N, max(1, N // 9))))
    tie_frames = tie_frames[::-1]
    for n, fr in enumerate(tie_frames):
        x[fr] = _frame_on_code(layers[0], targets[n % len(targets)], 1.0 + 0.1 * n)
    x = x.float()
    xb = x.reshape(B, T, 1024)
    q, idx, _, allq = rvq(xb.transpose(1, 2).contiguous().cuda())
    idx = idx.cpu().reshape(nq, N)
    ch = _Chain(layers, x.double())
    with torch.no_grad():
        _, io, _, _ = O.fvq_residual_vq([{k: v.double() for k, v in L.items()} for L in layers],
                                        xb.transpose(1, 2).double())
    for s in range(nq):                                   # the oracle's fvq chain is the same decision sequence
        assert torch.equal(io[s].reshape(N), ch.codes[s])
    lower = {a: a for a, _ in TIE_PAIRS}
    lower.update({b_: a for a, b_ in TIE_PAIRS})
    for n, fr in enumerate(tie_frames):
        j = targets[n % len(targets)]
        assert int(ch.codes[0][fr]) == lower[j]
        assert int(idx[0, fr]) == lower[j], f"frame {fr}: tie ({j}) resolved to {int(idx[0, fr])}"
    ok = ch.decidable()
    n_bad = int((~ok).sum())
    assert n_bad <= max(2, N // 5) + len(tie_frames)
    for s in range(nq):
        assert torch.equal(idx[s][ok], ch.codes[s][ok]), f"stage {s}"
    # quantized_out = x - final residual (one more rounding), for decidable frames within the chain's fp32 bound
    qf = q.cpu().transpose(1, 2).reshape(N, 1024).double()
    err = (qf - ch.qsum).abs()
    bound = ch.eps_r + U * ch.qsum.abs()
    assert (err[ok] <= bound[ok]).all()


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def _attention_ref(q, k, v, heads, vlen):
    """fp64 MultiHeadAttention.attention (modules/attentions.py:168-199): softmax(masked_fill(QK^T/16, mask, -1e4)) V on
    channels-last [B][T][heads*256]; returns o and the elementwise error bound of the fp32 kernels:
      score: 256 chained FMAs of q/16 (exact power-of-2 scale) -> |ds| <= gamma_256 sum_d |q_d k_d| / 16 + u|s|;
      the max shift: + u |s - max|;
      softmax: |dp_s| <= p_s (2 max|ds| + 8u + gamma_(T+64))  (exp and the reciprocal: a few roundings; the normaliser
      chains <= T/32 + 5 adds, plus <= 4 roundings per 32-key tile for the recomputing kernel's rescale);
      P V: <= T chained FMAs, so |do| <= (2 max|ds| + 8u + 2 gamma_(T+64)) sum_s p_s |v_s|."""
    B, T, C = q.shape
    qd, kd, vd = (t.double().reshape(B, T, heads, 256).transpose(1, 2) for t in (q, k, v))
    s = qd @ kd.transpose(-1, -2) / 16
    sabs = qd.abs() @ kd.abs().transpose(-1, -2) / 16
    if vlen is not None:
        valid = torch.arange(T)[None, :] < vlen[:, None]
        mask = valid[:, None, :, None] & valid[:, None, None, :]
        s = s.masked_fill(~mask, -1e4)
        sabs = sabs.masked_fill(~mask, 0.0)
    shift = (s - s.amax(-1, keepdim=True)).abs()
    ds = (gamma(256) * sabs + U * (s.abs() + shift).masked_fill(s == -1e4, 0.0)).amax(-1, keepdim=True)
    p = torch.softmax(s, -1)
    o = p @ vd
    bound = (2 * ds + 8 * U + 2 * gamma(T + 64)) * (p @ vd.abs())
    return (o.transpose(1, 2).reshape(B, T, C), bound.transpose(1, 2).reshape(B, T, C))


def _run_attention(q, k, v, heads, vlen, force_stream):
    e = _engine()
    B, T, C = q.shape
    qd, kd, vd = q.cuda(), k.cuda(), v.cuda()
    o = torch.full_like(qd, float("nan"))
    vl = vlen.to(torch.int32).cuda() if vlen is not None else None
    rc = e.L.fac_debug_attention(e.handle, _p(qd), _p(kd), _p(vd), _p(o), B, T, heads, _p(vl), force_stream, None)
    assert rc == 0, e.L.fac_last_error(e.handle)
    return o.cpu()


def _qkv(B, T, heads, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, T, heads * 256, generator=g) for _ in range(3)]     # scores ~ N(0, 1)


def _check_attention(o, ref, bound, vlen, v):
    assert torch.isfinite(o).all()
    err = (o.double() - ref).abs()
    assert (err <= bound).all(), f"max err {err.max():.3e}, max err/bound {(err / bound).max():.2f}"
    if vlen is not None:                       # masked queries: the mean of V over all T keys, as in the reference
        B, T, C = o.shape
        for b in range(B):
            if int(vlen[b]) < T:
                mean = v[b].double().mean(0)
                assert ((o[b, int(vlen[b]):].double() - mean).abs() <= bound[b, int(vlen[b]):]).all()


@pytest.mark.parametrize("force_stream", [0, 1])
@pytest.mark.parametrize("masked", [True, False])
@pytest.mark.parametrize("T", [1, 15, 16, 17, 31, 32, 33, 300])
def test_attention_vs_fp64(T, masked, force_stream, built_lib):
    """B = 3, heads = 2: the grid's y index b*heads + h must be split back into utterance and head; valid lengths 1,
    T - 1 and T in one batch."""
    B, heads = 3, 2
    q, k, v = _qkv(B, T, heads, T * 4 + masked * 2 + force_stream)
    vlen = torch.tensor([1, max(1, T - 1), T]) if masked else None
    ref, bound = _attention_ref(q, k, v, heads, vlen)
    o = _run_attention(q, k, v, heads, vlen, force_stream)
    _check_attention(o, ref, bound, vlen, v)


@pytest.mark.parametrize("T", [2430, 2431])
def test_attention_switch_between_kernels(T, built_lib):
    """launch_attention stores the [16][T] score block up to 200 KB of shared memory: T = 2430 uses exactly 204 800 bytes,
    T = 2431 recomputes the scores.  At 2431 the automatic choice must be the recomputing kernel, bit for bit."""
    B, heads = 2, 2
    q, k, v = _qkv(B, T, heads, T)
    vlen = torch.tensor([T, 1237])
    ref, bound = _attention_ref(q, k, v, heads, vlen)
    o = _run_attention(q, k, v, heads, vlen, 0)
    _check_attention(o, ref, bound, vlen, v)
    if T == 2431:
        assert torch.equal(o, _run_attention(q, k, v, heads, vlen, 1))


# ---------------------------------------------------------------------------------------------------------------------
# the masked timbre path end to end
# ---------------------------------------------------------------------------------------------------------------------
def _sd64(sd):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


def _style_encoder_frames(sd, mel, mask, prefix="timbre_encoder"):
    """O.style_encoder up to its fc layer: the per-frame outputs y [B][1024][T] that temporal_avg_pool sums."""
    from oracle import facodec_oracle as O
    x = F.conv1d(mel, sd[prefix + ".spectral.0.weight"], sd[prefix + ".spectral.0.bias"])
    x = O._mish(x)
    x = F.conv1d(x, sd[prefix + ".spectral.3.weight"], sd[prefix + ".spectral.3.bias"])
    x = O._mish(x) * mask
    x = O._conv1d_glu(x, sd, prefix + ".temporal.0")
    x = O._conv1d_glu(x, sd, prefix + ".temporal.1") * mask
    x = x + O._mha(x, sd, prefix + ".slf_attn", 2, mask.unsqueeze(2) * mask.unsqueeze(-1))
    return F.conv1d(x, sd[prefix + ".fc.weight"], sd[prefix + ".fc.bias"])


@pytest.mark.parametrize("T_full,lens", [
    (9137, (9137, 451, 5555)),               # full length; 300-599 samples (valid length 1); not a multiple of 300
    (2430 * 300, (2430 * 300, 700001)),      # 2430 mel frames: the stored-score attention kernel at its limit
    (2431 * 300 + 7, (2431 * 300 + 7, 12345)),   # 2431 mel frames: the recomputing attention kernel
])
def test_masked_timbre_vs_fp64(T_full, lens, built_lib):
    """timbre of m.quantizer(..., full_waves, wave_lens) vs O.quantizer_forward in fp64.
    temporal_avg_pool divides the sum over ALL T frames (masked frames are not zero after the attention's residual and
    fc's bias) by the valid length, so the error scale of utterance b is  mass_b = sum_t max_c |y_tc| / len_b  with y the
    fc output, not |timbre| (mass / |timbre| reaches ~60 for 41 valid frames of 2431).  Per frame, the StyleEncoder's
    seven convs run the promoted tensor-core class (each held to 4e-6 of its output's scale by test_gpu_kernels.py) and
    the attention is fp32-faithful (bounds above): 1e-5 of the frame's scale covers the chain; the pooled fp32 sum (four
    interleaved chains of T/4) adds gamma_(T/4+2).  |d timbre_bc| <= (1e-5 + gamma_(T/4+2)) mass_b.  The mask mistakes
    this test is after move timbre by O(|timbre|)."""
    from facodec_b200 import synth
    from conftest import state_dicts
    from oracle import facodec_oracle as O
    seed = 1
    m = _model(seed)
    sd = _sd64(state_dicts(seed)["quantizer"])
    B, T = len(lens), 1500
    x = synth.synth_waves(B, T, seed=T_full % 1000)
    full = synth.synth_waves(B, T_full, seed=T_full % 1000 + 1).squeeze(1)
    wl = torch.tensor(lens, dtype=torch.int64)
    g = torch.Generator().manual_seed(5)
    z = torch.randn(B, 1024, T // 300, generator=g)
    q = m.quantizer(z.cuda(), x.cuda(), n_c=2, full_waves=full.cuda(), wave_lens=wl.cuda())
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = O.quantizer_forward(sd, z.double(), x.double(), n_c=2, full_waves=full.double(), wave_lens=wl)[4]
        mel = O.mel_preprocess(sd, full.double().unsqueeze(1), n_bins=80)
        mask = O.sequence_mask(wl // 300, mel.size(-1)).unsqueeze(1)
        y = _style_encoder_frames(sd, mel, mask)
    Tm = mel.size(-1)
    mass = y.abs().amax(1).sum(1) / (wl // 300).double()                  # [B]
    bound = (1e-5 + gamma(Tm // 4 + 2)) * mass[:, None]
    err = (q[4].cpu().double() - ref).abs()
    print(f"TIMBRE T_full={T_full} lens={lens} maxerr={err.max():.3e} scale={ref.abs().max().item():.3f} "
          f"max err/bound={(err / bound).max():.3f}")
    assert (err <= bound).all(), f"max err/bound {(err / bound).max():.2f}"


# ---------------------------------------------------------------------------------------------------------------------
# mel front-end
# ---------------------------------------------------------------------------------------------------------------------
def _mel_ref(sd, wave):
    """fp64 O.mel_preprocess (n_bins = 80) and the elementwise bound of the fp32 kernels.
    Each DFT coefficient X = sum_j w_j x_j e^{-i theta} is one fp32 dot over the 1200 windowed samples: with the
    tensor-core class the basis is split into fp16 hi + 2^11-scaled fp16 lo (22 significant bits, u_eff = 2^-22) and
    summed in fp32 with promotion, with the fp32 FMA kernel u_eff = u; both are covered by
      |dRe|, |dIm| <= e = gamma_1200(u_eff = 2^-22) sum_j |w_j x_j|,  |d|X|^2| <= 2 sqrt2 |X| e + 2 e^2;
    the filterbank sum of 1025 non-negative terms adds gamma_1025 mel, and log / the affine map a few ulps:
      |d mel80| <= (sum_k fb_k |d|X_k|^2| + gamma_1025 mel) / (4 (1e-5 + mel)) + 4u (|log(1e-5 + mel)| + 4) / 4."""
    from oracle import facodec_oracle as O
    mel80 = O.mel_preprocess(sd, wave, n_bins=80)                       # [B][80][Tm]
    w = wave.squeeze(1)
    B, T = w.shape
    Tm = T // 300
    spec = torch.stft(w, 2048, hop_length=300, win_length=1200, window=sd["to_mel.spectrogram.window"], center=True,
                      pad_mode="reflect", normalized=False, onesided=True, return_complex=True)[..., :Tm]   # [B][1025][Tm]
    padded = F.pad(w[:, None], (1024, 1024), mode="reflect")[:, 0]
    frames = padded.unfold(1, 2048, 300)[:, :Tm, 424:424 + 1200]        # window centred in n_fft
    win = sd["to_mel.spectrogram.window"]
    sabs = (frames.abs() * win.abs()).sum(-1)                          # [B][Tm]
    ueff = 2.0 ** -22
    e = (1200 * ueff / (1 - 1200 * ueff)) * sabs
    dpow = 2 * math.sqrt(2) * spec.abs() * e[:, None, :] + 2 * e[:, None, :] ** 2
    fb = sd["to_mel.mel_scale.fb"]                                      # [1025][80]
    mel = torch.matmul(spec.abs().pow(2).transpose(1, 2), fb)           # [B][Tm][80]
    dmel = torch.matmul(dpow.transpose(1, 2), fb) + gamma(1025) * mel
    bound = dmel / (4 * (1e-5 + mel)) + 4 * U * ((torch.log(1e-5 + mel)).abs() + 4) / 4
    return mel80.transpose(1, 2), bound


@pytest.mark.parametrize("tensor_cores", [2, 1])
@pytest.mark.parametrize("T", [1025, 1200, 1499, 7201])
def test_mel80_vs_fp64(T, tensor_cores, built_lib):
    """T = 1025 is the shortest wave the centred reflect-padded STFT accepts (pad 1024 < T); 1499 and 7201 are not
    multiples of the hop; B = 3 checks the per-utterance offsets."""
    from facodec_b200 import synth
    from conftest import state_dicts
    seed = 1
    m = _model(seed)
    sd = _sd64(state_dicts(seed)["quantizer"])
    eng = m.quantizer._engine
    B, Tm = 3, T // 300
    x = synth.synth_waves(B, T, seed=T + 3)
    z = torch.randn(B, 1024, Tm + 1, generator=torch.Generator().manual_seed(T))
    tap = torch.full((B, Tm, 80), float("nan"), device="cuda")
    eng.set_option("tensor_cores", tensor_cores)
    try:
        eng.L.fac_debug_tap(eng.handle, b"mel80", _p(tap), tap.numel())
        m.quantizer(z.cuda(), x.cuda(), n_c=1)
        torch.cuda.synchronize()
    finally:
        eng.L.fac_debug_tap(eng.handle, b"mel80", None, 0)
        eng.set_option("tensor_cores", 2)
    ref, bound = _mel_ref(sd, x.double())
    got = tap.cpu().double()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    print(f"MEL T={T} tc={tensor_cores} maxerr={err.max():.3e} max err/bound={(err / bound).max():.3f}")
    assert (err <= bound).all(), f"max err {err.max():.3e}, max err/bound {(err / bound).max():.2f}"
