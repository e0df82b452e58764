"""The SLSTM recurrence kernels (lstm.cu, lstm2.cu) through fac_debug_slstm against a plain float64 loop.

slstm picks one of these routes (CONFIGS):

  name         hook / options                          recurrence                                input projection
  enc          upstream = 1                            lstm2, fp16 hi + 2^11-scaled lo, 3 passes promoted f16x2 (fp32-faithful)
  enc_v1       upstream = 1, lstm_v2 = 0               lstm.cu 3xTF32                            promoted f16x2
  dec          upstream = 0                            lstm2, ONE fp16 pass                      bf16 hi/lo, 3 products
  dec_v1       upstream = 0, decoder_lstm_fp16 = 0     lstm.cu bf16 hi/lo, 3 products            bf16 hi/lo
  dec_fp32     upstream = 0, decoder_bf16 = 0          lstm2 3-pass                              3xTF32
  dec_fp32_v1  upstream = 0, decoder_bf16 = 0, v2 = 0  lstm.cu 3xTF32                            3xTF32

The 3-pass resident pack does not fit in shared memory at H = 1536 (lstm2_smem_bytes > 227 KB), so enc and dec_fp32 run
lstm.cu's 3xTF32 kernel there, as the product does; lstm_rec2_kernel<12, true> is never launched.  Every other template
instantiation of both kernels runs in the short cases.

Bars.  y64 is the float64 loop, y32 the same loop in fp32, y_emul the float64 loop with the route's operand rounding.
  * enc, enc_v1: max|y - y64| <= max(16 max|y32 - y64|, 4e-6 max|y64|).  The first term scales with the run's own fp32
    error, so the bar holds where the cell state has long memory.  The factor is 16, not 4: the fp16 hi + scaled-lo pair and
    the 3xTF32 split carry 22 significant bits, not fp32's 24, so with both operands split the error can be 4-8x that of
    a plain fp32 loop (measured on an H100: 4.8x for enc in the integrating regime at T = 2400).
  * dec_fp32, dec_fp32_v1: the same with 160.  Their input projection is the non-promoted 3xTF32 conv class: its
    tensor-core accumulation truncates, so a small error of one sign enters every step's gates and the integrating cell
    state sums it (measured 36x the fp32 loop's error at H = 1024 and 84x at H = 1536, T = 400, in that regime; in the
    short cases these routes stay below 1/8 of the 4e-6 term).
  * dec (one fp16 pass): rms(y - y_emul) <= 0.5 rms(y_emul - y64) from T = 2 on, and
    max|y - y64| <= 1.5 max|y_emul - y64| + 4e-6 max|y64|.  The kernel differs from its rounding model by the fp32 rounding
    of y = h + x and of the gate math and by the truncating accumulation of the bf16 input projection; these are about a
    quarter of what the model's fp16 rounding moves (measured 0.15-0.26), and all of it at T = 1, where h_{-1} = 0 leaves
    no recurrent product to round.  Running the bf16 hi/lo class or 3-pass class instead gives a ratio near 1.
  * dec_v1 (bf16 hi/lo, 16 significant bits): max|y - y64| <= 4 max|y_emul - y64| + 4e-6 max|y64|.  Its rounding model is
    as small as the fp32 effects it leaves out (measured rms ratio 1.1-1.7), so no ratio is asserted for it.

Streaming carries (h, c) from one chunk to the next (LstmState): a chunked run must be bit-identical to the one-shot run,
because each row of the input projection is computed the same way whatever T is, and the carry copies fp32 c and the
published h words exactly.
"""
import ctypes
import math

import pytest
import torch

FAC_ERR_INVALID, FAC_ERR_UNSUPPORTED = -1, -4

# name -> (upstream, options, factor on the fp32 loop's error (fp32-grade routes), emulated (input projection, recurrence)
# rounding of the reduced-operand routes)
CONFIGS = {
    "enc": (1, {}, 16, None),
    "enc_v1": (1, {"lstm_v2": 0}, 16, None),
    "dec": (0, {}, None, ("bf16x3", "fp16")),
    "dec_v1": (0, {"decoder_lstm_fp16": 0}, None, ("bf16x3", "bf16x3")),
    "dec_fp32": (0, {"decoder_bf16": 0}, 160, None),
    "dec_fp32_v1": (0, {"decoder_bf16": 0, "lstm_v2": 0}, 160, None),
}
DEFAULT_OPTIONS = {"lstm_v2": 1, "decoder_lstm_fp16": 1, "decoder_bf16": 1}


# ---------------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------------
def f16_rn(v):
    """Round to the nearest fp16 (ties to even) through fp32, as the kernels round fp32 values."""
    return v.float().half().to(v.dtype)


def bf16_rn(v):
    """Round to the nearest bf16 (ties to even) through fp32."""
    return v.float().bfloat16().to(v.dtype)


def bf16_split(v):
    hi = bf16_rn(v)
    return hi, bf16_rn(v - hi)


def _mm(a, bt, mode):
    """a @ bt with the operands as one precision class sees them: None = exact, "fp16" = one pass over fp16_rn operands,
    "bf16x3" = a_hi b_hi + a_hi b_lo + a_lo b_hi with bf16 hi = rn(v), lo = rn(v - hi)."""
    if mode is None:
        return a @ bt
    if mode == "fp16":
        return f16_rn(a) @ f16_rn(bt)
    ah, al = bf16_split(a)
    bh, bl = bf16_split(bt)
    return ah @ bh + ah @ bl + al @ bh


def slstm_ref(x, ws, dtype=torch.float64, ih=None, rec=None):
    """SLSTM y = lstm2(lstm1(x)) + x (nn.LSTM(H, H, 2), gate order i, f, g, o, bias b_ih + b_hh, zero initial state) on
    x [B][T][H] in `dtype`, on x's device.  ih / rec emulate the operand rounding of the input projection / of W_hh and
    h_{t-1} (see _mm).  Returns y and the largest |c| and |gate pre-activation| seen."""
    B, T, H = x.shape
    inp = x.to(dtype)
    cmax = gmax = 0.0
    for l in range(2):
        w_ih, w_hh, b_ih, b_hh = (w.to(x.device, dtype) for w in ws[4 * l:4 * l + 4])
        xg = (_mm(inp.reshape(B * T, H), w_ih.t(), ih) + (b_ih + b_hh)).reshape(B, T, 4 * H)
        whT = w_hh.t().contiguous()
        if rec == "fp16":
            whT = f16_rn(whT)
        elif rec == "bf16x3":
            wh_hi, wh_lo = bf16_split(whT)
        h = torch.zeros(B, H, dtype=dtype, device=x.device)
        c = torch.zeros(B, H, dtype=dtype, device=x.device)
        out = torch.empty(B, T, H, dtype=dtype, device=x.device)
        cm = torch.zeros((), dtype=dtype, device=x.device)
        gm = torch.zeros((), dtype=dtype, device=x.device)
        for t in range(T):
            if rec is None:
                g = xg[:, t] + h @ whT
            elif rec == "fp16":
                g = xg[:, t] + f16_rn(h) @ whT
            else:
                hh, hl = bf16_split(h)
                g = xg[:, t] + hh @ wh_hi + hh @ wh_lo + hl @ wh_hi
            gi, gf, gg, go = g.chunk(4, dim=1)
            c = torch.sigmoid(gf) * c + torch.sigmoid(gi) * torch.tanh(gg)
            h = torch.sigmoid(go) * torch.tanh(c)
            out[:, t] = h
            cm = torch.maximum(cm, c.abs().max())
            gm = torch.maximum(gm, g.abs().max())
        cmax, gmax = max(cmax, cm.item()), max(gmax, gm.item())
        inp = out
    return inp + x.to(dtype), cmax, gmax


def test_reference_matches_torch_lstm_in_float64():
    """The fp64 loop without operand rounding is nn.LSTM(H, H, 2) + skip, in every regime."""
    for regime in REGIMES:
        H, B, T = 24, 3, 30
        ws = make_weights(H, regime)
        x = make_inputs(H, regime, B, T)
        lstm = torch.nn.LSTM(H, H, 2, batch_first=True).double()
        with torch.no_grad():
            for l in range(2):
                for i, n in enumerate(("weight_ih", "weight_hh", "bias_ih", "bias_hh")):
                    getattr(lstm, f"{n}_l{l}").copy_(ws[4 * l + i])
            ref = lstm(x.double())[0] + x.double()
        y, _, _ = slstm_ref(x, ws)
        assert (y - ref).abs().max().item() <= 1e-12 * max(1.0, ref.abs().max().item()), regime


@pytest.mark.parametrize("H", [1024, 1536])
def test_emulated_rounding_matches_the_packed_words(H, built_lib):
    """The emulation rounds W_hh exactly as the host packer does: fp16_rn is lstm2_pack's one-pass plane, bf16_split is
    lstm.cu's bf16 hi/lo words (fac_debug_lstm_pack modes 2 and 1)."""
    import numpy as np
    from facodec_b200 import _lib
    L = _lib.load()
    w = make_weights(H, "long_memory")[1].contiguous()
    wn = w.numpy()
    P = lambda a: ctypes.c_void_p(a.ctypes.data)
    info = (ctypes.c_int * 3)()
    n = L.fac_debug_lstm_pack(P(wn), H, 2, None, 0, info)
    U, G, R = info[0], info[1], info[2]
    words = np.zeros(n, np.float32)
    assert L.fac_debug_lstm_pack(P(wn), H, 2, P(words), n, info) == n
    wv = words.view(np.uint32).reshape(G, H // 16, 8, R)
    wr = w.reshape(4, G, U, H).permute(1, 0, 2, 3).reshape(G, R, H)                # [g][r = gate*U + u][k]
    q = f16_rn(wr).half().numpy().view(np.uint16)
    swz = (lambda k2: (k2 & 3) << 3) if R == 32 else (lambda k2: ((k2 >> 1) & 1) << 3)
    for k2 in range(8):
        wd = wv[:, :, k2, :][:, :, np.arange(R) ^ swz(k2)]                         # [g][sub][r]
        assert np.array_equal((wd & 0xFFFF).astype(np.uint16).transpose(0, 2, 1), q[:, :, 2 * k2::16])
        assert np.array_equal((wd >> 16).astype(np.uint16).transpose(0, 2, 1), q[:, :, 2 * k2 + 1::16])
    n = L.fac_debug_lstm_pack(P(wn), H, 1, None, 0, info)
    b = np.zeros(n, np.float32)
    assert L.fac_debug_lstm_pack(P(wn), H, 1, P(b), n, info) == n
    bw = b.view(np.uint32).reshape(G, H // 16, 2, 8, R)                              # [g][sub][hi|lo][k2][r]
    hi, lo = bf16_split(wr)
    for pl, ref in enumerate((hi, lo)):
        rb = (ref.float().numpy().view(np.uint32) >> 16).astype(np.uint16)           # bf16 bits (exact: ref is bf16)
        for k2 in range(8):
            wd = bw[:, :, pl, k2, :]
            assert np.array_equal((wd & 0xFFFF).astype(np.uint16).transpose(0, 2, 1), rb[:, :, 2 * k2::16])
            assert np.array_equal((wd >> 16).astype(np.uint16).transpose(0, 2, 1), rb[:, :, 2 * k2 + 1::16])


# ---------------------------------------------------------------------------------------------------------------------
# weight regimes and inputs
# ---------------------------------------------------------------------------------------------------------------------
# init:         every weight and bias uniform in +-1/sqrt(H) (nn.LSTM's default init, as synth._lstm), x ~ N(0, 1).
# long_memory:  forget-gate bias +4 (f ~ 0.98: memory of ~50 steps), x ~ 5 N(0, 1) so that layer-0 gate pre-activations
#               (std ~2.9) exceed 10 and saturate the gates.  W_hh keeps the init gain: at 3/sqrt(H) this recurrence is
#               chaotic (on an H100 the fp32 and fp64 loops differed by 0.65 at T = 400 and 1.9 at T = 2400, on outputs of
#               scale 25), which leaves no reference to hold a kernel to.
# integrating:  forget-gate bias +10 (f ~ 1 - 5e-5: c sums over thousands of steps) and x ~ N(0, 1) + 1: the constant
#               offset gives every unit a steady drive, so |c| drifts past 10 (fp32 c, tanhf at large arguments, expf at
#               both tails).
REGIMES = ("init", "long_memory", "integrating")
_WEIGHTS = {}


def make_weights(H, regime):
    key = (H, regime)
    if key not in _WEIGHTS:
        g = torch.Generator().manual_seed(1000 * H + REGIMES.index(regime))
        bound = 1.0 / math.sqrt(H)
        ws = []
        for _ in range(2):
            for shape in ((4 * H, H), (4 * H, H), (4 * H,), (4 * H,)):
                ws.append((torch.rand(shape, generator=g) * 2 - 1) * bound)
            if regime != "init":
                ws[-2][H:2 * H] += 4.0 if regime == "long_memory" else 10.0      # b_ih of the forget gate
        _WEIGHTS[key] = [w.contiguous() for w in ws]
    return _WEIGHTS[key]


def make_inputs(H, regime, B, T):
    g = torch.Generator().manual_seed(7 * H + 131 * B + T + 100000 * REGIMES.index(regime))
    x = torch.randn(B, T, H, generator=g)
    if regime == "long_memory":
        x = x * 5.0
    elif regime == "integrating":
        x = x + 1.0
    return x


# ---------------------------------------------------------------------------------------------------------------------
# GPU runs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engine(built_lib):
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    return e


def run_slstm(e, cfg, ws, x, chunks=None, fill=float("nan")):
    """fac_debug_slstm with the configuration's options (reset to the defaults afterwards).  x [B][T][H] on the GPU.
    Returns (status, y)."""
    upstream, opts, _, _ = CONFIGS[cfg]
    B, T, H = x.shape
    arr = (ctypes.c_void_p * 8)(*[w.data_ptr() for w in ws])
    y = torch.full_like(x, fill)
    ch = (ctypes.c_int * len(chunks))(*chunks) if chunks else None
    try:
        for k, v in opts.items():
            e.set_option(k, v)
        rc = e.L.fac_debug_slstm(e.handle, ctypes.c_void_p(x.data_ptr()), arr, B, T, H, upstream, ch,
                                 len(chunks) if chunks else 0, ctypes.c_void_p(y.data_ptr()), None)
    finally:
        for k in opts:
            e.set_option(k, DEFAULT_OPTIONS[k])
    torch.cuda.synchronize()
    return rc, y


_REFS = {}


def reference(H, regime, B, T, kind):
    """Cached reference on the GPU (cuBLAS float64 / float32 with TF32 off): kind = "64", "32" or an emulation pair."""
    key = (H, regime, B, T, kind)
    if key not in _REFS:
        if sum(r[0].numel() for r in _REFS.values()) > 2e8:
            _REFS.clear()
        x = make_inputs(H, regime, B, T).cuda()
        ws = make_weights(H, regime)
        tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            if kind == "32":
                _REFS[key] = slstm_ref(x, ws, torch.float32)
            elif kind == "64":
                _REFS[key] = slstm_ref(x, ws)
            else:
                _REFS[key] = slstm_ref(x, ws, ih=kind[0], rec=kind[1])
        finally:
            torch.backends.cuda.matmul.allow_tf32 = tf32
    return _REFS[key]


def check_against_reference(y, cfg, H, regime, tag, ref=None):
    """Holds the kernel's y [B][T][H] (GPU) to its route's bar; prints every error and ratio.  ref(kind) gives the
    reference for kind = "64", "32" or an emulation pair (slstm_ref's triple); by default the cached reference() of the
    regime's own weights and inputs."""
    B, T, _ = y.shape
    assert torch.isfinite(y).all(), f"{tag}: non-finite output"
    _, _, factor, emul = CONFIGS[cfg]
    if ref is None:
        ref = lambda kind: reference(H, regime, B, T, kind)
    y64, cmax, gmax = ref("64")
    yd = y.double()
    err = (yd - y64).abs().max().item()
    scale = y64.abs().max().item()
    if factor:
        y32 = ref("32")[0]
        err32 = (y32.double() - y64).abs().max().item()
        bar = max(factor * err32, 4e-6 * scale)
        print(f"LSTM {tag}: max|y-y64| {err:.3e}  max|y32-y64| {err32:.3e}  scale {scale:.2f}  bar {bar:.3e}  "
              f"ratio {err / bar:.3f}  max|c| {cmax:.1f}  max|gate| {gmax:.1f}")
        assert err <= bar, f"{tag}: max|y - y64| = {err:.3e} > {bar:.3e}"
    else:
        ye = ref(emul)[0]
        rms = lambda d: d.pow(2).mean().sqrt().item()
        d_kernel, d_model = rms(yd - ye), rms(ye - y64)
        err_e = (ye - y64).abs().max().item()
        one_pass = emul[1] == "fp16"
        bar = (1.5 if one_pass else 4.0) * err_e + 4e-6 * scale
        ratio = d_kernel / d_model if d_model > 0 else 0.0
        print(f"LSTM {tag}: rms(y-y_emul) {d_kernel:.3e}  rms(y_emul-y64) {d_model:.3e}  ratio {ratio:.4f}  "
              f"max|y-y64| {err:.3e}  max|y_emul-y64| {err_e:.3e}  bar {bar:.3e}  scale {scale:.2f}  max|c| {cmax:.1f}  "
              f"max|gate| {gmax:.1f}")
        if one_pass and T > 1:
            assert d_kernel <= 0.5 * d_model, f"{tag}: rms(y - y_emul) = {d_kernel:.3e} > 0.5 x {d_model:.3e}"
        assert err <= bar, f"{tag}: max|y - y64| = {err:.3e} > {bar:.3e}"
    return cmax, gmax


def _check_one_shot(engine, cfg, H, regime, B, T):
    ws = make_weights(H, regime)
    x = make_inputs(H, regime, B, T).cuda()
    rc, y = run_slstm(engine, cfg, ws, x)
    assert rc == 0, engine.L.fac_last_error(engine.handle)
    return check_against_reference(y, cfg, H, regime, f"{cfg} {regime} H={H} B={B} T={T}")


SHORT_SHAPES = [(B, T, H) for H in (1024, 1536) for B in (1, 5, 32) for T in (1, 2, 3, 40)] + \
               [(2, 5, 1024), (3, 17, 1536), (32, 4, 1024), (5, 40, 1536)]
# at H = 1536 enc_v1 is enc and dec_fp32 is dec_fp32_v1 (no 3-pass resident pack): those are run once
SHORT_CASES = [(cfg, B, T, H) for cfg in CONFIGS for (B, T, H) in SHORT_SHAPES
               if not (H == 1536 and cfg in ("enc_v1", "dec_fp32"))]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,B,T,H", SHORT_CASES)
def test_slstm_short(cfg, B, T, H, engine):
    """Every route at both widths, single-step and two-step sequences (the parity slots of the h exchange), a batch of one,
    a partial batch tile and a full one."""
    _check_one_shot(engine, cfg, H, "init", B, T)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [33, 65])
@pytest.mark.parametrize("cfg,H", [("enc", 1024), ("dec", 1536)])
def test_slstm_more_than_32_sequences(cfg, H, B, engine):
    """Above 32 sequences slstm makes one launch per 32, all sharing the h exchange, hT and barrier scratch."""
    _check_one_shot(engine, cfg, H, "long_memory", B, 50)


# The long_memory regime runs 400 frames only: by 2400 frames its fp32 and fp64 loops differ by 1.6 on outputs of scale 25
# (measured on an H100), so there is nothing left to compare a kernel with.
LONG_CASES = [(cfg, H, T, regime) for cfg, H in (("enc", 1024), ("dec", 1536))
              for T, regime in ((2400, "integrating"), (400, "long_memory"))] + \
             [(cfg, H, 400, regime) for cfg, H in (("enc_v1", 1024), ("dec_v1", 1536), ("dec_fp32", 1024), ("dec_fp32_v1", 1536))
              for regime in ("long_memory", "integrating")]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,H,T,regime", LONG_CASES)
def test_slstm_long(cfg, H, T, regime, engine):
    """Long sequences with trained-like memory: 2400 frames is 30 s of audio.  Errors that add up in c over hundreds of
    steps show here and not in the short cases."""
    cmax, gmax = _check_one_shot(engine, cfg, H, regime, 2, T)
    if regime == "integrating":
        assert cmax > 10.0, "the integrating regime must drive |c| past 10"
    else:
        assert gmax > 10.0, "the long-memory regime must saturate some gates"


CHUNK_LISTS = [[1, 1, 1, 37], [2, 3, 5, 7, 11, 13], [6, 300, 1, 93]]


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 31, 32])
@pytest.mark.parametrize("cfg,H", [("enc", 1024), ("dec", 1024), ("dec", 1536)])
def test_slstm_chunked_state_carry_is_bit_exact(cfg, H, B, engine):
    """The streamed state carry: chunks of one frame and of odd and even lengths (both parity slots of the h exchange end a
    chunk) must give exactly the one-shot output.  The one-shot run over 400 frames is held to the bars; its first
    40 / 41 frames are those of one-shot runs over 40 / 41 frames, for the same reason chunking is exact.  (The encoder's
    3-pass recurrence has no resident-W pack at H = 1536, so it cannot stream there: see the error-path test.)"""
    regime = "long_memory"
    ws = make_weights(H, regime)
    x = make_inputs(H, regime, B, 400).cuda()
    rc, y_full = run_slstm(engine, cfg, ws, x)
    assert rc == 0, engine.L.fac_last_error(engine.handle)
    for chunks in CHUNK_LISTS:
        T = sum(chunks)
        rc, y = run_slstm(engine, cfg, ws, x[:, :T].contiguous(), chunks)
        assert rc == 0, engine.L.fac_last_error(engine.handle)
        diff = (y - y_full[:, :T]).abs()
        bad = (diff > 0) | ~torch.isfinite(y)
        first = bad.nonzero()[0].tolist() if bad.any() else None
        print(f"LSTM chunked {cfg} H={H} B={B} chunks={chunks}: differing values {int(bad.sum())}, "
              f"max diff {diff.max().item():.3e}, first at [b, t, j] = {first}")
        assert not bad.any(), f"chunks {chunks}: output differs from the one-shot run, first at [b, t, j] = {first}"
    check_against_reference(y_full, cfg, H, regime, f"{cfg} {regime} H={H} B={B} T=400 one-shot")


@pytest.mark.gpu
def test_slstm_chunked_error_paths(engine):
    """Chunked runs that cannot stream or whose chunk list is wrong return their status and write nothing."""
    def expect(rc_want, cfg, H, B, T, chunks, what):
        ws = make_weights(H, "init")
        x = make_inputs(H, "init", B, T).cuda()
        rc, y = run_slstm(engine, cfg, ws, x, chunks)
        assert rc == rc_want, f"{what}: status {rc}, expected {rc_want}"
        assert torch.isnan(y).all(), f"{what}: the output was written"
    expect(FAC_ERR_UNSUPPORTED, "enc", 1024, 33, 4, [2, 2], "B = 33 chunked")
    expect(FAC_ERR_UNSUPPORTED, "dec", 1024, 33, 4, [2, 2], "B = 33 chunked")
    expect(FAC_ERR_UNSUPPORTED, "enc_v1", 1024, 2, 4, [2, 2], "lstm_v2 = 0 chunked")
    expect(FAC_ERR_UNSUPPORTED, "dec_v1", 1536, 2, 4, [2, 2], "decoder_lstm_fp16 = 0 chunked")
    expect(FAC_ERR_UNSUPPORTED, "enc", 1536, 2, 4, [2, 2], "3-pass recurrence at H = 1536 chunked")
    expect(FAC_ERR_INVALID, "enc", 1024, 2, 6, [2, 2], "chunks sum to 4, T = 6")
    expect(FAC_ERR_INVALID, "dec", 1536, 2, 4, [2, 0, 2], "zero-length chunk")
    expect(FAC_ERR_INVALID, "dec", 1024, 2, 4, [3, 2, -1], "negative chunk")
