"""Sessions at other sample rates in the stream pools (CodecStreamPool, VoiceConversionPool, CodecDecodePool): each one equals
the 24 kHz offline call composed with resample(), bit for bit, while 24 kHz sessions sharing its steps stay equal to their
own B = 1 streams, and a pool of 24 kHz sessions runs the same launches as before."""
import random

import pytest
import torch

import facodec_b200 as fb
from facodec_b200 import _lib

RATES = [16000, 44100, 48000, 24000, 24000]


def _models():
    from test_gpu_parity import model_for, redec_model_for
    return model_for(0), redec_model_for(0)


def _wave(T, seed):
    from facodec_b200 import synth
    return synth.synth_waves(1, T, seed=seed).cuda()


def _cat_codes(parts):
    return [torch.cat([p[k] for p in parts], dim=2) for k in range(3)]


@pytest.mark.gpu
def test_codec_stream_pool_rates(built_lib):
    codec, _ = _models()
    rng = random.Random(11)
    pool = fb.CodecStreamPool(codec, capacity=8, n_c=2)
    secs = [1.3, 0.9, 1.1, 1.2, 0.8]
    xs = [_wave(int(r * s), 100 + i) for i, (r, s) in enumerate(zip(RATES, secs))]
    joins = [0, 1, 0, 2, 0]
    sess, pos, parts, done = {}, {}, {i: [] for i in range(len(RATES))}, {}
    step = 0
    while len(done) < len(RATES):
        chunks = {}
        for i, r in enumerate(RATES):
            if i in done or step < joins[i]:
                continue
            if i not in sess:
                sess[i] = pool.open(sample_rate=r)
                pos[i] = 0
            T = xs[i].shape[-1]
            if r == 24000:
                k = 3000 if pos[i] == 0 else 300 * rng.randint(1, 8)
            else:
                k = rng.choice([0, 1, int(0.25 * r), 2205, 5000])
            k = min(k, T - pos[i])
            if r == 24000 and (k < 300 or (pos[i] == 0 and k < 3000)):
                continue
            if r == 24000:
                k -= k % 300
            chunks[sess[i]] = xs[i][:, :, pos[i]:pos[i] + k]
            pos[i] += k
        if chunks:
            out = pool.encode_codes(chunks)
            for i, s in sess.items():
                if i not in done and s in out:
                    parts[i].append(out[s])
        ending = [i for i in sess if i not in done and (xs[i].shape[-1] - pos[i] < (300 if RATES[i] == 24000 else 1))
                  and pos[i] > 0]
        if ending:
            fin = pool.finish_codes([sess[i] for i in ending])
            for i in ending:
                codes, timbre = fin[sess[i]]
                parts[i].append(codes)
                done[i] = timbre
                pool.close(sess[i])
        step += 1
    for i, r in enumerate(RATES):
        codes = _cat_codes(parts[i])
        rx = fb.resample(xs[i], r, 24000)
        L = pos[i] if r == 24000 else rx.shape[-1] // 300 * 300
        ref, timbre = fb.Codec(codec).encode(rx[..., :L], n_c=2)
        for a, b in zip(codes, ref):
            assert torch.equal(a, b), (r, a.shape, b.shape)
        assert torch.equal(done[i], timbre), r
    pool.close()


@pytest.mark.gpu
def test_codec_stream_pool_short_rate_session(built_lib):
    codec, _ = _models()
    pool = fb.CodecStreamPool(codec, capacity=2)
    s = pool.open(sample_rate=48000)
    assert pool.encode_codes({s: _wave(4000, 1)})[s][0].shape == (1, 1, 0)
    with pytest.raises(_lib.FacError):
        pool.finish_codes([s])                         # 2000 samples at 24 kHz
    with pytest.raises(ValueError):
        pool.open(sample_rate=7000)
    pool.close()


def _codes(T, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 1024, (1, r, T), generator=g).cuda() for r in (1, 2, 3)]


@pytest.mark.gpu
def test_voice_conversion_pool_rates(built_lib):
    codec, rm = _models()
    vc = fb.VoiceConverter(rm)
    pool = fb.VoiceConversionPool(rm, capacity=8)
    rng = random.Random(5)
    Ts = [70, 90, 60, 80, 75]
    codes = [_codes(T, 200 + i) for i, T in enumerate(Ts)]
    timbres = [torch.randn(1, 1024, generator=torch.Generator().manual_seed(i)).cuda() for i in range(len(Ts))]
    sess, owner, finished = {}, {}, set()
    outs = {i: [] for i in range(len(Ts))}
    pos = [0] * len(Ts)
    joins = [0, 2, 1, 0, 3]
    step = 0
    while len(finished) < len(Ts):
        chunks = {}
        for i, T in enumerate(Ts):
            if step < joins[i] or pos[i] >= T:
                continue
            if i not in sess:
                sess[i] = pool.open(timbres[i], sample_rate=RATES[i])
                owner[sess[i]] = i
            F = min(rng.randint(1, 20), T - pos[i])
            chunks[sess[i]] = [c[:, :, pos[i]:pos[i] + F] for c in codes[i][:2]]
            pos[i] += F
        if chunks:
            for s, y in pool.convert(chunks).items():
                outs[owner[s]].append(y.view(-1))
        ending = [i for i in sess if pos[i] >= Ts[i] and i not in finished]
        if ending:
            for s, y in pool.finish([sess[i] for i in ending]).items():
                outs[owner[s]].append(y.view(-1))
            for i in ending:
                finished.add(i)
                pool.close(sess[i])
        step += 1
    for i, r in enumerate(RATES):
        got = torch.cat(outs[i])
        ref = vc.convert(codes[i], timbres[i])
        if r != 24000:
            ref = fb.resample(ref, 24000, r)
        assert torch.equal(got, ref.view(-1)), r
    pool.close()


@pytest.mark.gpu
def test_decode_pool_rates_and_launches(built_lib):
    codec, _ = _models()
    pool = fb.CodecDecodePool(codec, capacity=8)
    plain = fb.CodecDecodePool(codec, capacity=8)
    rng = random.Random(9)
    Ts = [40, 50, 45, 60, 35]
    codes = [_codes(T, 300 + i) for i, T in enumerate(Ts)]
    timbres = [torch.randn(1, 1024, generator=torch.Generator().manual_seed(10 + i)).cuda() for i in range(len(Ts))]
    sess = [pool.open(timbres[i], sample_rate=r) for i, r in enumerate(RATES)]
    outs = {i: [] for i in range(len(Ts))}
    refs = {i: [] for i in range(len(Ts))}
    streams = [fb.CodecStream(codec, 1) for _ in Ts]
    pos = [0] * len(Ts)
    while any(p < T for p, T in zip(pos, Ts)):
        chunks, sizes = {}, {}
        for i, T in enumerate(Ts):
            if pos[i] >= T:
                continue
            F = min(10 if pos[i] == 0 else rng.randint(1, 12), T - pos[i])
            sizes[i] = F
            chunks[sess[i]] = [c[:, :, pos[i]:pos[i] + F] for c in codes[i]]
            pos[i] += F
        got = pool.decode_codes(chunks)
        for i in sizes:
            outs[i].append(got[sess[i]].view(-1))
            refs[i].append(streams[i].decode_codes(chunks[sess[i]], timbres[i]).view(-1))
    fin = pool.finish(sess)
    for i, r in enumerate(RATES):
        ref = torch.cat(refs[i]).view(1, 1, -1)
        if r != 24000:
            ref = fb.resample(ref, 24000, r)
        else:
            assert fin[sess[i]].numel() == 0
        assert torch.equal(torch.cat(outs[i] + [fin[sess[i]].view(-1)]), ref.view(-1)), r
        streams[i].close()
    # a step of 24 kHz sessions only runs the launches of a pool that never had a rate session
    a = pool.open(timbres[0])
    b = plain.open(timbres[0])
    c0 = codes[0]
    ya = pool.decode_codes({a: c0})[a]
    na = fb.Codec(codec).launch_count()
    yb = plain.decode_codes({b: c0})[b]
    nb = fb.Codec(codec).launch_count()
    assert na == nb and torch.equal(ya, yb)
    pool.close()
    plain.close()
