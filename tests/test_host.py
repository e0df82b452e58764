"""CPU: host-side logic and the C-ABI surface (no compute calls without a GPU)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT


def _declared(header):
    hdr = open(os.path.join(ROOT, "include", header)).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(fac_[a-z_0-9]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol(built_lib):
    """include/facodec_b200.h is the drop-in surface (SURVEY.md 8b) and holds no test hook; the kernel-level hooks and
    the profiling calls live in include/facodec_b200_debug.h.  Every symbol either header declares is exported."""
    public, debug = _declared("facodec_b200.h"), _declared("facodec_b200_debug.h")
    assert len(public) >= 15
    assert not [n for n in public if n.startswith(("fac_debug_", "fac_profile_"))]
    assert all(n.startswith(("fac_debug_", "fac_profile_")) for n in debug)
    lib = ctypes.CDLL(built_lib)
    for name in public + debug:
        assert hasattr(lib, name), f"{name} declared in include/ but not exported"
    from facodec_b200 import _lib
    assert sorted(_lib.EXPORTED) == sorted(public + debug)
    L = _lib.load()
    assert L.fac_abi_version() == 2


def test_encode_frames_matches_reference_rule(built_lib):
    """ceil(T / 300) for the causal strided stack (encodec.py:71-78 extra padding)."""
    from facodec_b200 import _lib
    L = _lib.load()
    for T in (300, 900, 1500, 7000, 7200, 96000, 96001, 12345):
        t = T
        for s in (2, 5, 5, 6):
            t = -(-t // s)
        assert L.fac_encode_frames(T) == t


def test_no_gpu_fails_loudly(built_lib):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import facodec_b200 as fb
    model = fb.build_model()
    for m in model.values():
        m.eval()
    with pytest.raises(fb.FacError):
        model.encoder(torch.zeros(1, 1, 3000))


def test_state_dict_surface_matches_reference_keys():
    import facodec_b200 as fb
    from facodec_b200 import synth
    model = fb.build_model()
    sds = synth.synth_state_dicts(0)
    for name in ("encoder", "quantizer", "decoder"):
        sd = model[name].state_dict()
        assert list(sd.keys()) == list(sds[name].keys())
        for k in sd:
            assert tuple(sd[k].shape) == tuple(sds[name][k].shape)
        model[name].load_state_dict(sds[name])
        assert torch.equal(model[name].state_dict()["%s" % list(sd.keys())[3]], sds[name][list(sd.keys())[3]])
        bad = dict(sds[name])
        bad.pop(next(iter(bad)))
        with pytest.raises(RuntimeError):
            model[name].load_state_dict(bad)
    assert sum(p.numel() for p in model.encoder.parameters()) == 36283520
    assert sum(p.numel() for p in model.decoder.parameters()) == 85536866
    with pytest.raises(NotImplementedError):
        model.encoder.train()
        model.encoder(torch.zeros(1, 1, 3000))


def test_build_model_accepts_reference_config():
    import yaml
    import facodec_b200 as fb
    cfg = yaml.safe_load("""
model_params:
  causal: True
  lstm: 2
  separate_prosody_encoder: True
  n_c_codebooks: 2
  timbre_norm: True
  DAC: {encoder_dim: 64, encoder_rates: [2, 5, 5, 6], decoder_dim: 1536, decoder_rates: [6, 5, 5, 2], sr: 24000}
""")
    m = fb.build_model(cfg["model_params"])
    assert set(m.keys()) == {"encoder", "quantizer", "decoder"}
    assert m.encoder._engine is m.decoder._engine is m.quantizer._engine
    with pytest.raises(NotImplementedError):
        fb.build_model({"causal": False})


def test_mel_buffers_close_to_torchaudio():
    import torchaudio
    from facodec_b200 import synth
    fb = synth.melscale_fbanks_htk()
    ref = torchaudio.functional.melscale_fbanks(1025, 0.0, 12000.0, 80, 24000, norm=None, mel_scale="htk")
    assert (fb - ref).abs().max() < 2e-5
    assert (synth.hann_window_periodic(1200) - torch.hann_window(1200)).abs().max() < 5e-7


def test_shard_range_partitions():
    from facodec_b200.distributed import shard_range
    for n in (0, 1, 7, 32, 256, 257):
        for w in (1, 2, 3, 8):
            spans = [shard_range(n, r, w) for r in range(w)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(spans[i][1] == spans[i + 1][0] for i in range(w - 1))
            sizes = [b - a for a, b in spans]
            assert max(sizes) - min(sizes) <= 1


def _plan(L, Cin, Cout, K, dil, stride, Tout, mode, occ2):
    import ctypes
    out = (ctypes.c_int * 8)()
    rc = L.fac_debug_tc_plan(Cin, Cout, K, dil, stride, Tout, mode, occ2, out)
    return rc, dict(zip(("N", "MT", "nchunk", "stages", "rows", "smem", "Rpad", "promote_every"), list(out)))


SMEM_CAP = 227 * 1024     # dynamic shared memory per block on sm_90


def _check_plan(p, Cout, mode, K, stride):
    """A plan the wgmma kernel can run: N | Cout in 16-channel steps, a tile of 128 rows (warpgroups split rows) or 64 rows
    (they split channels), per-warpgroup accumulators of <= 128 floats (<= 64 when promoted: master + window registers),
    1-2 weight stages, shared memory within the SM, promotion windows of <= 48 chained MMAs."""
    assert Cout % p["N"] == 0 and p["N"] % 16 == 0
    assert p["rows"] == 64 * p["MT"] and p["MT"] in (1, 2)
    nw = p["N"] if p["MT"] == 2 else p["N"] // 2
    assert nw % 16 == 0 and nw <= (64 if mode in (1, 3) else 128)
    assert 1 <= p["stages"] <= 2 and p["smem"] <= SMEM_CAP
    if mode in (1, 3):
        Kr = K if stride == 1 else 2
        assert p["promote_every"] * Kr * (1 if mode == 3 else 6) <= 48 or p["promote_every"] == 1


def test_tensor_core_tile_plans_respect_hardware_limits(built_lib):
    """Host logic of the tensor-core path (no GPU): every layer geometry of the model gets a plan inside the SM's limits
    (_check_plan) and ineligible layers are refused."""
    from facodec_b200 import _lib
    L = _lib.load()
    enc = [(64, 64, 7, d, 1, 96000) for d in (1, 3, 9)] + [(128, 128, 7, 9, 1, 48000), (256, 256, 7, 9, 1, 9600),
           (512, 512, 7, 9, 1, 1920), (64, 128, 4, 1, 2, 48000), (128, 256, 10, 1, 5, 9600), (256, 512, 10, 1, 5, 1920),
           (512, 1024, 12, 1, 6, 320), (1024, 1024, 3, 1, 1, 320), (1024, 4096, 1, 1, 1, 10240), (1200, 2176, 1, 1, 1, 10240),
           (256, 512, 5, 1, 1, 320), (512, 1024, 5, 1, 1, 320)]
    for (Cin, Cout, K, dil, stride, T) in enc:
        for mode in (1, 3):
            rc, p = _plan(L, Cin, Cout, K, dil, stride, T, mode, 0)
            assert rc == 0, (Cin, Cout, K, mode)
            _check_plan(p, Cout, mode, K, stride)
    dec = [(1024, 1536, 7, 1, 1, 320), (1536, 6144, 1, 1, 1, 10240), (768, 768, 7, 9, 1, 1920), (384, 384, 7, 3, 1, 9600),
           (384, 384, 1, 1, 1, 9600), (192, 192, 2, 1, 1, 48000), (1536, 4608, 2, 1, 1, 320)]
    for (Cin, Cout, K, dil, stride, T) in dec:
        rc, p = _plan(L, Cin, Cout, K, dil, stride, T, 2, 0)
        assert rc == 0
        _check_plan(p, Cout, 2, K, stride)
    # fused ResidualUnits keep every channel in one tile: N = C
    for C in (96, 192, 256):
        rc, p = _plan(L, C, C, 7, 9, 1, 48000, 4, 0)
        assert rc == 0 and p["N"] == C
        _check_plan(p, C, 4, 7, 1)
    # not eligible: Cin not a multiple of 16 per row, odd strides, fused with Cin != Cout
    assert _plan(L, 20, 256, 1, 1, 1, 320, 1, 0)[0] != 0
    assert _plan(L, 64, 64, 7, 1, 3, 100, 0, 0)[0] != 0
    assert _plan(L, 96, 192, 7, 1, 1, 100, 4, 0)[0] != 0


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("geom", [(64, 64, 7, 1), (128, 256, 10, 5), (96, 96, 1, 1), (32, 48, 3, 1)])
def test_tensor_core_weight_blob_layout_and_split(geom, mode, built_lib):
    """Host logic (no GPU): the tensor-core weight blob.  Decodes [ntile][chunk][tap][hi|lo][k-group][N][16 B] back to W and
    checks the split classes: TF32 pair / bf16 pair / fp16 hi + 2^11-scaled lo reconstruct w to their mantissa budget
    and each half is exactly representable in its format."""
    import ctypes
    import numpy as np
    from facodec_b200 import _lib
    L = _lib.load()
    Cin, Cout, K, stride = geom
    rng = np.random.RandomState(Cin + Cout + K)
    w = (rng.randn(Cout, Cin, K) / np.sqrt(Cin * K)).astype(np.float32)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)
    n = L.fac_debug_tc_pack(P(w), Cin, Cout, K, stride, mode, None, 0)
    if n < 0:
        pytest.skip("geometry not eligible in this mode")
    blob = np.zeros(n, np.float32)
    assert L.fac_debug_tc_pack(P(w), Cin, Cout, K, stride, mode, P(blob), n) == n
    out = (ctypes.c_int * 8)()
    assert L.fac_debug_tc_plan(Cin, Cout, K, 1, stride, 0, mode, 0, out) == 0
    N, nchunk = out[0], out[2]
    Kr, vf = (K, 1) if stride == 1 else (2, stride)
    # generic row-tap matrix the kernels contract over: Wg[tap][j][co], j = (sample-in-row, ci)
    Wg = np.zeros((Kr, vf * Cin, Cout), np.float32)
    for k in range(K):
        Wg[k // vf, (k % vf) * Cin:(k % vf + 1) * Cin, :] = w[:, :, k].T
    nt = Cout // N
    if mode in (0, 1):
        b = blob.reshape(nt, nchunk, Kr, 2, 4, N, 4)                 # [..][hl][k4][n][e]
        hi = b[:, :, :, 0].transpose(0, 1, 2, 4, 3, 5).reshape(nt, nchunk, Kr, N, 16)
        lo = b[:, :, :, 1].transpose(0, 1, 2, 4, 3, 5).reshape(nt, nchunk, Kr, N, 16)
        assert not (hi.view(np.uint32) & 0x1FFF).any() and not (lo.view(np.uint32) & 0x1FFF).any()   # exact TF32
        rec, tol = hi.astype(np.float64) + lo, 2.0 ** -20
    else:
        h16 = blob.view(np.uint16).reshape(nt, nchunk, Kr, 2, 2, N, 8)  # [..][hl][k8][n][e]
        def dec(a):
            a = a.transpose(0, 1, 2, 4, 3, 5).reshape(nt, nchunk, Kr, N, 16)
            if mode == 2:
                return (a.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
            return a.view(np.float16).astype(np.float64)
        hi, lo = dec(np.ascontiguousarray(h16[:, :, :, 0])), dec(np.ascontiguousarray(h16[:, :, :, 1]))
        rec = hi + (lo / 2048.0 if mode == 3 else lo)
        tol = 2.0 ** -15 if mode == 2 else 2.0 ** -20
    # rec[nt][chunk][tap][n][kk] == Wg[tap][chunk*16 + kk][nt*N + n]
    ref = Wg.reshape(Kr, nchunk, 16, nt, N).transpose(3, 1, 0, 4, 2)
    err = np.abs(rec - ref).max()
    assert err <= tol * np.abs(ref).max(), (err, tol)


@pytest.mark.parametrize("L,pl,pr", [(300, 6, 0), (40, 54, 0), (5, 6, 0), (7, 6, 2), (1, 6, 0), (55, 54, 3), (9000, 600, 600), (3, 18, 5)])
def test_pad_index_map_matches_reference_pad1d(L, pl, pr, built_lib):
    """Host logic (no GPU): the reflect-padding index map of the kernels == encodec.py:96-113 pad1d, including the
    branch that zero-extends inputs shorter than the padding before reflecting (oracle restatement, pinned to the
    reference by test_oracle.py)."""
    import ctypes
    import torch
    from facodec_b200 import _lib
    from oracle import facodec_oracle as O
    Lb = _lib.load()
    n = pl + L + pr
    out = (ctypes.c_int * n)()
    assert Lb.fac_debug_pad_map(L, pl, pr, 1, out, n) == 0
    ramp = torch.arange(1, L + 1, dtype=torch.float32).view(1, 1, L)      # value i+1 marks source row i; 0 = zero fill
    ref = O._pad1d_reflect(ramp, pl, pr).view(-1)
    got = torch.tensor([0.0 if s < 0 else float(s + 1) for s in out])
    assert torch.equal(got, ref)
    assert Lb.fac_debug_pad_map(L, pl, pr, 0, out, n) == 0                  # zero padding
    assert [s for s in out] == [-1] * pl + list(range(L)) + [-1] * pr


@pytest.mark.parametrize("H", [1024, 1536])
def test_lstm_recurrent_weight_packing(H, built_lib):
    """Host logic (no GPU): W_hh [4H][H] -> per-CTA slices.  fp32 layout: CTA g holds rows gate*U + u = W[gate*H + g*U + u]
    as [k][4U]; bf16 layout: the same slice as hi/lo words of two consecutive k (hi + lo reproduces w to 2^-16)."""
    import ctypes
    import numpy as np
    from facodec_b200 import _lib
    L = _lib.load()
    rng = np.random.RandomState(H)
    w = (rng.uniform(-1, 1, size=(4 * H, H)) / np.sqrt(H)).astype(np.float32)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)
    info = (ctypes.c_int * 3)()
    n = L.fac_debug_lstm_pack(P(w), H, 0, None, 0, info)
    U, G, R = info[0], info[1], info[2]
    assert n == G * H * R and G * U == H and R == 4 * U and G <= 132
    f = np.zeros(n, np.float32)
    assert L.fac_debug_lstm_pack(P(w), H, 0, P(f), n, info) == n
    f = f.reshape(G, H, 4, U)                                              # [g][k][gate][u]
    ref = w.reshape(4, G, U, H).transpose(1, 3, 0, 2)                      # W[gate*H + g*U + u][k] -> [g][k][gate][u]
    assert np.array_equal(f, ref)
    b = np.zeros(n, np.float32)
    assert L.fac_debug_lstm_pack(P(w), H, 1, P(b), n, info) == n
    words = b.view(np.uint32).reshape(G, H // 16, 2, 8, R)                 # [g][sub][hl][k2][r]
    def bf(x):
        return (x.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    lo_half, hi_half = words & 0xFFFF, words >> 16                         # even k in the low half
    val = np.stack([bf(lo_half), bf(hi_half)], axis=-1)                    # [g][sub][hl][k2][r][parity]
    rec = val[:, :, 0] + val[:, :, 1]                                      # hi + lo -> [g][sub][k2][r][parity]
    rec = rec.transpose(0, 1, 2, 4, 3).reshape(G, H, R)                    # k = sub*16 + 2*k2 + parity
    ref2 = ref.reshape(G, H, R).astype(np.float64)
    assert np.abs(rec - ref2).max() <= 2.0 ** -16 * np.abs(ref2).max()


def test_header_is_plain_c_and_links_from_c(built_lib, tmp_path):
    """The boundary is a C ABI: include/facodec_b200.h must compile as C99 and a C program must be able to link the
    library and call it (host-only entry points, so this runs without a GPU)."""
    import os
    import shutil
    import subprocess
    from facodec_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = _lib.lib_path()
    src = tmp_path / "abi.c"
    src.write_text(r'''
#include <stdio.h>
#include "facodec_b200.h"
#include "facodec_b200_debug.h"
int main(void) {
    int plan[8];
    int pad[9];
    if (fac_abi_version() != 2) return 2;
    if (fac_debug_tc_plan(192, 192, 7, 9, 1, 48000, 4, 0, plan) != FAC_OK) return 3;
    if (fac_debug_pad_map(3, 6, 0, 1, pad, 9) != FAC_OK) return 4;
    if (fac_encode_frames(96000) != 320) return 5;
    printf("%d %d %d %d\n", plan[0], plan[1], plan[4], pad[0]);
    return 0;
}
''')
    exe = tmp_path / "abi"
    cmd = [gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", str(exe), lib,
           "-Wl,-rpath," + os.path.dirname(lib)]
    subprocess.check_call(cmd)
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64:" + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.check_output([str(exe)], env=env, text=True).split()
    assert out[:3] == ["192", "1", "64"]         # fused C = 192 unit: N = 192, warpgroups split channels, 64-row tiles


@pytest.mark.parametrize("H,mode", [(1024, 3), (1024, 2), (1536, 2)])
def test_lstm2_resident_weight_words(H, mode, built_lib):
    """Host logic (no GPU): lstm2.cu's resident W_hh layout -- fp16 pairs of consecutive k per 32-bit word, XOR-swizzled
    columns -- holds round-to-nearest fp16 planes bit for bit (the rounding test_gpu_lstm.py's emulation assumes), decodes
    back to W_hh (one pass: fp16 rounding 2^-11; three-pass: hi + lo'/2^11 to 2^-20), and every
    mma.sync fragment load (4 k pairs x 8 rows per instruction) touches 32 distinct shared-memory banks."""
    import ctypes
    import numpy as np
    from facodec_b200 import _lib
    L = _lib.load()
    rng = np.random.RandomState(H + mode)
    w = (rng.uniform(-1, 1, size=(4 * H, H)) / np.sqrt(H)).astype(np.float32)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)
    info = (ctypes.c_int * 3)()
    n = L.fac_debug_lstm_pack(P(w), H, mode, None, 0, info)
    U, G, R = info[0], info[1], info[2]
    PL = 2 if mode == 3 else 1
    assert n == G * (H // 16) * PL * 8 * R
    words = np.zeros(n, np.float32)
    assert L.fac_debug_lstm_pack(P(w), H, mode, P(words), n, info) == n
    wv = words.view(np.uint32).reshape(G, H // 16, PL, 8, R)
    swz = (lambda k2: (k2 & 3) << 3) if R == 32 else (lambda k2: ((k2 >> 1) & 1) << 3)
    w32 = w.reshape(4, G, U, H).transpose(1, 0, 2, 3).reshape(G, R, H)                        # [g][r = gate*U + u][k]
    ref = w32.astype(np.float64)
    # the planes bit for bit: hi = rn_f16(w), lo' = rn_f16((w - hi) * 2^11) (numpy's float16 casts round to nearest even)
    hi_ref = w32.astype(np.float16)
    planes = [hi_ref, ((w32 - hi_ref.astype(np.float32)) * np.float32(2048)).astype(np.float16)]
    rec = np.zeros((G, R, H))
    for k2 in range(8):
        cols = np.arange(R) ^ swz(k2)
        for pl in range(PL):
            wd = wv[:, :, pl, k2, :][:, :, cols]                                               # [g][sub][r]
            lo16 = (wd & 0xFFFF).astype(np.uint16).view(np.float16)
            hi16 = (wd >> 16).astype(np.uint16).view(np.float16)
            assert np.array_equal(lo16.transpose(0, 2, 1).view(np.uint16), planes[pl][:, :, 2 * k2::16].view(np.uint16))
            assert np.array_equal(hi16.transpose(0, 2, 1).view(np.uint16), planes[pl][:, :, 2 * k2 + 1::16].view(np.uint16))
            sc = 1.0 if pl == 0 else 1.0 / 2048.0
            rec[:, :, 2 * k2::16] += sc * lo16.astype(np.float64).transpose(0, 2, 1)
            rec[:, :, 2 * k2 + 1::16] += sc * hi16.astype(np.float64).transpose(0, 2, 1)
    tol = 2.0 ** -20 if mode == 3 else 2.0 ** -11
    assert np.abs(rec - ref).max() <= tol * np.abs(ref).max()
    # bank check of one A-fragment load instruction: lanes (fg = row 0..7, ft = k pair 0..3) -> word address ft*R + (row ^ swz)
    for i in range(R // 16):
        for half in (0, 8):
            banks = {((ft * R) + ((i * 16 + fg + half) ^ swz(ft))) % 32 for fg in range(8) for ft in range(4)}
            assert len(banks) == 32


@pytest.mark.parametrize("stride", [2, 5, 6])
def test_transposed_conv_as_conv_causal_and_noncausal(stride, built_lib):
    """Host logic (no GPU): ConvTranspose1d(k = 2s, stride s) + the reference's trims (encodec.py:248-270) == a 2-tap
    (causal) / 3-tap (non-causal) zero-padded conv with s*Cout phase-major channels, checked against the oracle's
    sconvtr1d (pinned to the imported reference)."""
    import ctypes
    import numpy as np
    import torch
    import torch.nn.functional as F
    from facodec_b200 import _lib
    from oracle import facodec_oracle as O
    L = _lib.load()
    Cin, Cout, T = 6, 4, 9
    g = torch.Generator().manual_seed(stride)
    w = torch.randn(Cin, Cout, 2 * stride, generator=g)
    x = torch.randn(2, Cin, T, generator=g)
    sd = {"c.weight": w, "c.bias": torch.zeros(Cout)}
    P = lambda a: ctypes.c_void_p(a.ctypes.data)
    wn = np.ascontiguousarray(w.numpy())
    for causal in (1, 0):
        n = L.fac_debug_convtr_pack(P(wn), Cin, Cout, stride, causal, None, 0)
        taps = 2 if causal else 3
        assert n == taps * Cin * stride * Cout
        pk = np.zeros(n, np.float32)
        assert L.fac_debug_convtr_pack(P(wn), Cin, Cout, stride, causal, P(pk), n) == n
        wk = torch.from_numpy(pk.reshape(taps, Cin, stride * Cout)).permute(2, 1, 0).contiguous()   # conv1d weight [s*Cout][Cin][taps]
        xp = F.pad(x, (1, 0 if causal else 1))
        y = F.conv1d(xp, wk)                                                    # [B][s*Cout][T], channel r*Cout + co
        y = y.view(2, stride, Cout, T).permute(0, 2, 3, 1).reshape(2, Cout, T * stride)
        ref = O.sconvtr1d(x, sd, "c", stride, causal=bool(causal))
        assert ref.shape == y.shape
        assert float((y - ref).abs().max()) <= 1e-5


def test_dac_code_file_round_trip(tmp_path):
    """facodec_b200.codefile (dac/model/base.py:15-54 format) without the reference: round trip, uint16 range check,
    version check, the [p | c | r] codebook order."""
    import numpy as np
    import pytest
    import torch
    from facodec_b200 import codefile
    g = torch.Generator().manual_seed(1)
    codes = [torch.randint(0, 1024, (3, n, 11), generator=g) for n in (1, 1, 3)]
    f = codefile.from_forward(codes, original_length=3300)
    p = f.save(tmp_path / "x.anything")
    assert p.name == "x.dac"
    raw = np.load(p, allow_pickle=True)[()]
    assert raw["codes"].dtype == np.uint16 and raw["codes"].shape == (3, 5, 11)
    assert set(raw["metadata"]) == {"input_db", "original_length", "sample_rate", "chunk_length", "channels", "padding", "dac_version"}
    back = codefile.DACFile.load(p)
    for u, v in zip(codefile.unpack_codes(back.codes, n_c=1), codes):
        assert torch.equal(u, v)
    with pytest.raises(ValueError):
        codefile.from_forward([torch.full((1, 1, 2), 70000)] * 3, 600).save(tmp_path / "big")
    raw["metadata"]["dac_version"] = "9.9"
    with open(tmp_path / "bad.dac", "wb") as fh:
        np.save(fh, raw)
    with pytest.raises(RuntimeError):
        codefile.DACFile.load(tmp_path / "bad.dac")
    with pytest.raises(ValueError):
        codefile.unpack_codes(back.codes, n_c=2)


def test_fa_predictors_state_dict_surface():
    """facodec_b200.FApredictors (modules/quantize.py:456-619) without a GPU: the reference's key set (heads of the reversal
    predictors at index 1 of their nn.Sequential, the Linear timbre predictor under timbre_norm), load/save round trip,
    CPU tensors refused."""
    import pytest
    import torch
    import facodec_b200 as fb
    m = fb.FApredictors(in_dim=32, timbre_norm=True, use_gr_content_global_f0=True, use_gr_residual_f0=True, use_gr_residual_phone=True,
                        use_gr_x_timbre=True, n_speakers=50).eval()
    sd = m.state_dict()
    tops = {k.split(".model.")[0].split(".heads.")[0] for k in sd if ".model." in k or ".heads." in k}
    assert tops == {"f0_predictor", "phone_predictor", "rev_f0_predictor.1", "rev_content_predictor.1", "rev_timbre_predictor.1",
                    "rev_global_f0_predictor.1"}
    assert sd["timbre_predictor.weight"].shape == (50, 32) and sd["global_f0_predictor.weight"].shape == (1, 32)
    assert sd["f0_predictor.heads.1.weight"].shape == (1, 32) and sd["phone_predictor.heads.0.weight"].shape == (1024, 32)
    sd2 = {k: v + 1 for k, v in sd.items()}
    m.load_state_dict(sd2)
    assert torch.equal(m.state_dict()["timbre_predictor.bias"], sd2["timbre_predictor.bias"])
    assert torch.equal(m.state_dict()["rev_f0_predictor.1.heads.0.weight"], sd2["rev_f0_predictor.1.heads.0.weight"])
    with pytest.raises(fb.FacError):
        m([torch.zeros(1, 32, 5)] * 3, torch.zeros(1, 32))


def test_tile_plans_of_every_codec_layer_fit_the_sm(built_lib):
    """Host logic (no GPU): the tensor-core tile plans of every conv geometry of config.yml's encoder (promoted, fp16 hi +
    scaled-lo split) and decoder (bf16 split / fused units) at the benchmark lengths stay inside one SM (_check_plan)."""
    import ctypes
    from facodec_b200 import _lib
    L = _lib.load()
    out = (ctypes.c_int * 8)()
    keys = ("N", "MT", "nchunk", "stages", "rows", "smem", "Rpad", "promote_every")
    enc = []                                    # (Cin, Cout, K, dil, stride, Tout)
    T, c = 96000, 64
    for s in (2, 5, 5, 6):
        for d in (1, 3, 9):
            enc += [(c, c, 7, d, 1, T), (c, c, 1, 1, 1, T)]
        enc.append((c, 2 * c, 2 * s, 1, s, T // s))
        T //= s
        c *= 2
    enc += [(1024, 4096, 1, 1, 1, 320 * 32), (1024, 1024, 3, 1, 1, 320)]
    for (ci, co, k, d, st, to) in enc:
        assert L.fac_debug_tc_plan(ci, co, k, d, st, to, 3, 0, out) == 0, (ci, co, k)
        _check_plan(dict(zip(keys, list(out))), co, 3, k, st)
    dec = []
    T, c = 320, 1536
    for s in (6, 5, 5, 2):
        dec.append((c, (c // 2) * s, 2, 1, 1, T, 2))                 # transposed conv as a 2-tap conv with s * Cout channels
        T *= s
        c //= 2
        for d in (1, 3, 9):
            if c <= 256:
                dec.append((c, c, 7, d, 1, T, 4))                    # fused ResidualUnit
            else:
                dec += [(c, c, 7, d, 1, T, 2), (c, c, 1, 1, 1, T, 2)]
    dec += [(1024, 1536, 7, 1, 1, 320, 2), (1536, 6144, 1, 1, 1, 320 * 32, 2)]
    for (ci, co, k, d, st, to, mode) in dec:
        assert L.fac_debug_tc_plan(ci, co, k, d, st, to, mode, 0, out) == 0, (ci, co, k, mode)
        _check_plan(dict(zip(keys, list(out))), co, mode, k, st)
