"""The sinc resampler on the GPU (fac_resample, fac_rs_pool_*; facodec_b200.resample, ResamplePool): offline outputs
against the fp64 restatement, ragged lanes against their own B = 1 calls, and streams against the offline call bit for
bit, whatever the chunking."""
import ctypes
import random

import pytest
import torch

import facodec_b200 as fb
from facodec_b200 import _lib
from facodec_b200.modules import _rs_engine, _rs_geometry
from oracle.resample import resample64

RATES = [8000, 11025, 16000, 22050, 32000, 44100, 48000, 96000, 192000]
PAIRS = [(r, 24000) for r in RATES if r != 24000] + [(24000, r) for r in RATES if r != 24000]


def _x(B, T, seed):
    return torch.randn(B, T, generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("orig,new", PAIRS)
def test_offline_within_fp64_bound(orig, new, built_lib):
    o, n, width, K = _rs_geometry(orig, new)
    for T in (1, max(width - 1, 1), K - 1, 4801):
        x = _x(3, T, T + orig)
        y = fb.resample(x, orig, new)
        y64, mass = resample64(x, o, n, width, fb.resample_table(orig, new))
        assert y.shape == y64.shape
        err = (y.cpu().double() - y64).abs()
        assert bool((err <= (K + 1) * 2.0 ** -24 * mass).all()), (T, float(err.max()))


@pytest.mark.gpu
@pytest.mark.parametrize("orig,new", [(44100, 24000), (24000, 48000), (24000, 11025)])
def test_against_torchaudio_on_gpu(orig, new, built_lib):
    """torchaudio on the same GPU with TF32 convolutions off (cuDNN would otherwise round the taps to TF32); its table is
    built with CUDA sin / cos, so it agrees within the fp32 bound rather than bit for bit."""
    F = pytest.importorskip("torchaudio.functional")
    o, n, width, K = _rs_geometry(orig, new)
    x = _x(2, 24001, 3)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        ta = F.resample(x, orig, new)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    y64, mass = resample64(x, o, n, width, fb.resample_table(orig, new))
    assert ta.shape == fb.resample(x, orig, new).shape
    assert bool(((ta.cpu().double() - y64).abs() <= 4 * (K + 1) * 2.0 ** -24 * mass + 1e-6).all())


@pytest.mark.gpu
def test_shapes_and_equal_rates(built_lib):
    x = _x(2, 1000, 1)
    assert fb.resample(x.view(2, 1, 1000), 44100, 24000).shape == (2, 1, 545)
    assert torch.equal(fb.resample(x, 24000, 24000), x)
    with pytest.raises(ValueError):
        fb.resample(x, 7000, 24000)
    with pytest.raises(_lib.FacError):
        fb.resample(x.cpu(), 44100, 24000)


@pytest.mark.gpu
@pytest.mark.parametrize("orig,new", [(44100, 24000), (24000, 44100), (16000, 24000), (24000, 8000)])
def test_ragged_lanes_equal_b1(orig, new, built_lib):
    T = 3001
    lens = [T, 1, 17, 1500, 0, 2999]
    x = _x(len(lens), T, 9)
    y = fb.resample(x, orig, new, lengths=lens)
    for b, n in enumerate(lens):
        m = fb.resample_length(orig, new, n)
        if n:
            assert torch.equal(y[b, :m], fb.resample(x[b:b + 1, :n], orig, new)[0])
        assert bool((y[b, m:] == 0).all())


@pytest.mark.gpu
def test_every_output_written_once(built_lib):
    """A NaN-prefilled output buffer comes back without a NaN: every sample, tails included, is written."""
    e = _rs_engine(torch.device("cuda"))
    fb.resample(_x(1, 10, 0), 44100, 24000)            # registers the table
    x = _x(4, 5000, 2)
    Tout = fb.resample_length(44100, 24000, 5000)
    y = torch.full((4, Tout), float("nan"), device="cuda")
    lens = (ctypes.c_int * 4)(5000, 3, 0, 4321)
    rc = e.L.fac_resample(e.handle, ctypes.c_void_p(x.data_ptr()), 4, 5000, lens, 44100, 24000, ctypes.c_void_p(y.data_ptr()),
                          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(e.handle, rc, "fac_resample")
    assert not bool(y.isnan().any())
    assert torch.equal(y, fb.resample(x, 44100, 24000, lengths=[5000, 3, 0, 4321]))


def _chunks(T, rng):
    cuts, p = [], 0
    while p < T:
        k = rng.choice([0, 1, 1, 2, 7, 300, 523, 1103, 2205, 4410])
        k = min(k, T - p)
        cuts.append((p, p + k))
        p += k
    cuts.insert(rng.randrange(len(cuts) + 1), (p, p))
    return cuts


@pytest.mark.gpu
@pytest.mark.parametrize("quantum", [1, 300])
@pytest.mark.parametrize("orig,new", PAIRS)
def test_stream_equals_offline(orig, new, quantum, built_lib):
    rng = random.Random(orig * 7 + new + quantum)
    pool = fb.ResamplePool(4, quantum=quantum)
    for T in (1, 700, 9001):
        x = _x(1, T, T)
        s = pool.open(orig, new)
        outs = []
        for a, b in _chunks(T, rng):
            y = pool.push({s: x[:, a:b]})[s]
            assert y.shape[2] % quantum == 0
            outs.append(y.view(-1))
        outs.append(pool.finish([s])[s].view(-1))
        assert torch.equal(torch.cat(outs), fb.resample(x, orig, new)[0]), (T,)
        pool.close(s)
    pool.close()


@pytest.mark.gpu
def test_mixed_rates_in_one_step_equal_alone(built_lib):
    """Sessions of different pairs stepped together equal each stepped alone; a slot closed mid-stream and reopened at
    another pair starts clean; the finish can carry a last chunk."""
    pairs = [(48000, 24000), (24000, 48000), (44100, 24000), (24000, 11025), (16000, 24000), (24000, 24000)]
    rng = random.Random(3)
    T = 12000
    xs = [_x(1, T, 40 + i) for i in range(len(pairs))]
    cuts = [_chunks(T, rng) for _ in pairs]
    shared = fb.ResamplePool(8, quantum=300)
    ss = [shared.open(*p) for p in pairs]
    stale = shared.open(44100, 24000)
    shared.push({stale: _x(1, 5000, 99)})
    shared.close(stale)
    outs = [[] for _ in pairs]
    for step in range(max(len(c) for c in cuts)):
        chunks = {ss[i]: xs[i][:, a:b] for i, c in enumerate(cuts) if step < len(c) for a, b in [c[step]]}
        for s, y in shared.push(chunks).items():
            outs[ss.index(s)].append(y.view(-1))
    re = shared.open(8000, 24000)                      # the closed slot, reopened at another pair
    xr = _x(1, 4000, 77)
    tail = shared.finish({ss[i]: None if i % 2 else xs[i][:, :0] for i in range(len(pairs))})
    r = torch.cat([shared.push({re: xr[:, :1234]})[re].view(-1), shared.finish({re: xr[:, 1234:]})[re].view(-1)])
    assert torch.equal(r, fb.resample(xr, 8000, 24000)[0])
    for i, p in enumerate(pairs):
        alone = fb.ResamplePool(1, quantum=300)
        s = alone.open(*p)
        ref = [alone.push({s: xs[i][:, a:b]})[s].view(-1) for a, b in cuts[i]] + [alone.finish([s])[s].view(-1)]
        got = torch.cat(outs[i] + [tail[ss[i]].view(-1)])
        assert torch.equal(got, torch.cat(ref)), p
        assert torch.equal(got, fb.resample(xs[i], *p)[0]), p
        alone.close()
    shared.close()


@pytest.mark.gpu
def test_rejected_step_leaves_state(built_lib):
    pool = fb.ResamplePool(3)
    a, b = pool.open(44100, 24000), pool.open(24000, 48000)
    x = _x(1, 6000, 5)
    ya = pool.push({a: x[:, :2000], b: x[:, :2000]})
    with pytest.raises(_lib.FacError):
        pool.push({a: x[:, 2000:4000], 7: x[:, :10]})               # 7 is not open
    with pytest.raises(ValueError):
        pool.push({a: x[:, 2000:4000], b: x.view(1, 1, 1, -1)})     # bad shape
    fin = pool.finish([b])
    with pytest.raises(_lib.FacError):
        pool.push({a: x[:, 2000:4000], b: x[:, :5]})                 # b is finished: the whole step is rejected
    ra = torch.cat([ya[a].view(-1), pool.push({a: x[:, 2000:]})[a].view(-1), pool.finish([a])[a].view(-1)])
    assert torch.equal(ra, fb.resample(x, 44100, 24000)[0])
    assert torch.equal(torch.cat([ya[b].view(-1), fin[b].view(-1)]), fb.resample(x[:, :2000], 24000, 48000)[0])
    pool.close()
