"""A rejected step of a pool that holds sessions at other sample rates leaves every session as it was: the resampler step
is checked before it runs, or taken back when the encoder rejects the step, and a decode-pool session that finish() ended
is refused before the decoder runs."""
import pytest
import torch

import facodec_b200 as fb
from facodec_b200 import _lib


def _models():
    from test_gpu_parity import model_for
    return model_for(0)


def _wave(T, seed):
    from facodec_b200 import synth
    return synth.synth_waves(1, T, seed=seed).cuda()


def _codes(T, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 1024, (1, r, T), generator=g).cuda() for r in (1, 2, 3)]


def _expect(codec, x48, parts, timbre):
    r = fb.resample(x48, 48000, 24000)
    L = r.shape[-1] // 300 * 300
    ref, t = fb.Codec(codec).encode(r[..., :L], n_c=2)
    codes = [torch.cat([p[k] for p in parts], dim=2) for k in range(3)]
    for a, b in zip(codes, ref):
        assert torch.equal(a, b)
    assert torch.equal(timbre, t)


@pytest.mark.gpu
def test_finished_24k_session_beside_48k_session(built_lib):
    codec = _models()
    pool = fb.CodecStreamPool(codec, capacity=4, n_c=2)
    a, b = pool.open(), pool.open(sample_rate=48000)
    x24, x48 = _wave(6000, 1), _wave(30000, 2)
    parts = [pool.encode_codes({a: x24[..., :3000], b: x48[..., :7000]})[b]]
    pool.finish_codes([a])                                  # finished, not closed
    with pytest.raises(_lib.FacError):
        pool.encode_codes({a: x24[..., 3000:], b: x48[..., 7000:15000]})
    with pytest.raises(_lib.FacError):
        pool.finish_codes([a, b])
    parts.append(pool.encode_codes({b: x48[..., 7000:15000]})[b])
    parts.append(pool.encode_codes({b: x48[..., 15000:]})[b])
    codes, timbre = pool.finish_codes([b])[b]
    _expect(codec, x48, parts + [codes], timbre)
    pool.close()


@pytest.mark.gpu
def test_encoder_rejection_takes_the_resampler_step_back(built_lib):
    """A rule only the encoder checks (here: compression needs tensor_cores = 2) rejects the step after the resampler ran:
    the resampler sessions get their samples back."""
    codec = _models()
    e = codec.encoder._engine
    pool = fb.CodecStreamPool(codec, capacity=4, n_c=2)
    b = pool.open(sample_rate=48000)
    x48 = _wave(30000, 3)
    parts = [pool.encode_codes({b: x48[..., :9000]})[b]]
    e.set_option("tensor_cores", 1)
    try:
        with pytest.raises(_lib.FacError):
            pool.encode_codes({b: x48[..., 9000:20000]})
        with pytest.raises(_lib.FacError):
            pool.finish_codes([b])
    finally:
        e.set_option("tensor_cores", 2)
    parts.append(pool.encode_codes({b: x48[..., 9000:20000]})[b])
    parts.append(pool.encode_codes({b: x48[..., 20000:]})[b])
    codes, timbre = pool.finish_codes([b])[b]
    _expect(codec, x48, parts + [codes], timbre)
    pool.close()


@pytest.mark.gpu
def test_decode_pool_refuses_finished_session(built_lib):
    codec = _models()
    pool = fb.CodecDecodePool(codec, capacity=4)
    timbre = torch.randn(1, 1024, generator=torch.Generator().manual_seed(4)).cuda()
    f, g = pool.open(timbre, sample_rate=48000), pool.open(timbre)
    cf, cg = _codes(30, 5), _codes(40, 6)
    ref = fb.CodecStream(codec, 1)
    want = [ref.decode_codes([c[..., :12] for c in cg], timbre).view(-1)]
    got = [pool.decode_codes({f: [c[..., :12] for c in cf], g: [c[..., :12] for c in cg]})[g].view(-1)]
    pool.finish([f])
    with pytest.raises(_lib.FacError):
        pool.decode_codes({f: [c[..., 12:20] for c in cf], g: [c[..., 12:20] for c in cg]})
    with pytest.raises(_lib.FacError):
        pool.finish([f])
    got.append(pool.decode_codes({g: [c[..., 12:] for c in cg]})[g].view(-1))
    want.append(ref.decode_codes([c[..., 12:] for c in cg], timbre).view(-1))
    assert torch.equal(torch.cat(got), torch.cat(want))
    ref.close()
    pool.close(f)
    f2 = pool.open(timbre, sample_rate=16000)               # the slot, reopened, starts clean
    y = torch.cat([pool.decode_codes({f2: cf})[f2].view(-1), pool.finish([f2])[f2].view(-1)])
    s = fb.CodecStream(codec, 1)
    assert torch.equal(y, fb.resample(s.decode_codes(cf, timbre), 24000, 16000).view(-1))
    s.close()
    pool.close()


@pytest.mark.gpu
def test_resample_pool_undo(built_lib):
    pool = fb.ResamplePool(2, quantum=300)
    s = pool.open(44100, 24000)
    x = torch.randn(1, 20000, generator=torch.Generator().manual_seed(7)).cuda()
    out = [pool.push({s: x[:, :5000]})[s].view(-1)]
    pool.push({s: x[:, 5000:9000]})
    pool._undo([s])
    with pytest.raises(_lib.FacError):
        pool._undo([s])                                     # one step back only
    out.append(pool.push({s: x[:, 5000:12000]})[s].view(-1))
    pool.finish({s: x[:, 12000:]})
    pool._undo([s])
    out.append(pool.finish({s: x[:, 12000:]})[s].view(-1))
    assert torch.equal(torch.cat(out), fb.resample(x, 44100, 24000)[0])
    pool.close()
