"""The timbre without the rest of the encode, and before the end of a live utterance.

* Codec.timbre (fac_codec_timbre_lens): Codec.encode's timbre bit for bit from the mel front-end and the StyleEncoder alone.
* CodecStream.timbre (fac_stream_timbre): the timbre finish_codes() would return if the utterance ended now, i.e.
  Codec.encode's on every sample fed so far, without ending the stream or changing anything it emits later.
* CodecStreamPool.timbre (fac_codes_pool_timbre): the same for many sessions in shared ragged StyleEncoder batches, each
  its own B = 1 stream's.
* CodecDecodePool.set_timbre (fac_dec_pool_set_timbre): a receiver switching voice between chunks, equal to a B = 1
  CodecStream.decode_codes given the new timbre from that chunk on.
On the host: the pool's batch plan against a restatement.  On the GPU: every equality above, with torch.equal."""
import ctypes
import random

import pytest
import torch

from conftest import GOLDEN_CASES, case_inputs, state_dicts

HOP, LANE_MAX, FRAME_BUDGET = 300, 32, 1 << 15


def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    new = ("fac_codec_timbre_lens", "fac_stream_timbre", "fac_codes_pool_timbre", "fac_dec_pool_set_timbre")
    assert set(new) <= set(_declared("facodec_b200.h"))
    assert "fac_debug_timbre_plan" in _declared("facodec_b200_debug.h")
    assert set(new) | {"fac_debug_timbre_plan"} <= set(_lib.EXPORTED)


# ---------------------------------------------------------------------------------------------------------------------
# host: the batch plan of CodecStreamPool.timbre
# ---------------------------------------------------------------------------------------------------------------------
def _plan_engine(frames):
    from facodec_b200 import _lib
    L = _lib.load()
    n = len(frames)
    batch = (ctypes.c_int * max(n, 1))()
    nb = L.fac_debug_timbre_plan(n, (ctypes.c_int * max(n, 1))(*frames), batch)
    assert nb >= 0
    return list(batch)[:n], nb


def _plan_restated(frames):
    """Sessions by frame count (stable); a batch takes the next while it has < 32 lanes and lanes x longest stays within
    the frame budget."""
    batches = []
    for i in sorted(range(len(frames)), key=lambda i: frames[i]):
        if not batches or len(batches[-1]) == LANE_MAX or (len(batches[-1]) + 1) * frames[i] > FRAME_BUDGET:
            batches.append([])
        batches[-1].append(i)
    batch = [0] * len(frames)
    for k, b in enumerate(batches):
        for i in b:
            batch[i] = k
    return batch, len(batches)


@pytest.mark.parametrize("seed", range(6))
def test_timbre_plan_matches_restatement(seed, built_lib):
    rng = random.Random(seed)
    n = rng.choice([1, 7, 40, 130])
    frames = [rng.choice([10, rng.randint(10, 400), rng.randint(400, 5000), rng.randint(5000, 300000)]) for _ in range(n)]
    batch, nb = _plan_engine(frames)
    assert (batch, nb) == _plan_restated(frames)
    for k in range(nb):
        lanes = [frames[i] for i in range(n) if batch[i] == k]
        assert 1 <= len(lanes) <= LANE_MAX
        assert len(lanes) == 1 or len(lanes) * max(lanes) <= FRAME_BUDGET
    assert _plan_engine([]) == ([], 0)


def test_timbre_plan_bounds_an_hour_long_caller(built_lib):
    """32 callers of 3 s share one batch; beside an hour-long caller (288 000 frames), that one runs alone."""
    short = [240] * 32
    assert _plan_engine(short)[1] == 1
    batch, nb = _plan_engine(short + [288000])
    assert nb == 2 and batch[-1] == 1 and set(batch[:-1]) == {0}
    batch, nb = _plan_engine([4800] * 32)                 # 60 s each: 6 lanes per batch
    assert nb == 6 and max(batch.count(k) for k in range(nb)) == 6


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _model(seed=1):
    from test_gpu_parity import model_for
    return model_for(seed)


def _waves(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 1, T, generator=g) * 0.1).to("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(1, 9000), (3, 20000), (2, 1025)])
def test_codec_timbre_equals_encode(B, T, built_lib):
    import facodec_b200 as fb
    codec = fb.Codec(_model())
    x = _waves(B, T, 40 + B)
    t = codec.timbre(x)
    n_t = codec.launch_count()
    for n_c in (1, 2):
        _, ref = codec.encode(x, n_c)
        assert torch.equal(t, ref), n_c
    n_enc = codec.launch_count()
    print("launches: Codec.timbre %d, Codec.encode %d" % (n_t, n_enc))
    assert 0 < n_t < n_enc


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(n for n, c in GOLDEN_CASES.items() if "full" not in c))
def test_codec_timbre_golden_shapes(name, built_lib):
    import facodec_b200 as fb
    c = GOLDEN_CASES[name]
    from test_gpu_parity import model_for
    codec = fb.Codec(model_for(c["wseed"]))
    x, _ = case_inputs(c)
    x = x.to("cuda:0")
    assert torch.equal(codec.timbre(x), codec.encode(x, c["n_c"])[1])


@pytest.mark.gpu
def test_codec_timbre_lengths(built_lib):
    """Each lane of a ragged call equals the ragged encode's timbre and its own B = 1 call."""
    import facodec_b200 as fb
    codec = fb.Codec(_model())
    x = _waves(4, 24000, 9)
    lens = [24000, 7301, 1025, 15000]
    t = codec.timbre(x, lengths=lens)
    assert torch.equal(t, codec.encode(x, 2, lengths=lens)[1])
    assert torch.equal(t, codec.timbre(x, lengths=torch.tensor(lens)))
    for b, n in enumerate(lens):
        assert torch.equal(t[b:b + 1], codec.timbre(x[b:b + 1, :, :n].contiguous())), b
    with pytest.raises(ValueError):
        codec.timbre(x, lengths=[24000, 1024, 3000, 3000])     # as Codec.encode: lengths in (1024, T]
    with pytest.raises(ValueError):
        codec.timbre(x, lengths=[24000, 3000])
    with pytest.raises(fb.FacError):
        codec.timbre(x.cpu())


@pytest.mark.gpu
def test_codec_timbre_vs_fp64(built_lib):
    """The oracle's fp64 style_encoder(mel_preprocess(x)), held to the bound of the masked timbre test
    (test_gpu_quantizer_kernels.py): |d timbre| <= (1e-5 + gamma_(T/4+2)) mass with mass = sum_t max_c |y_tc| / T."""
    import facodec_b200 as fb
    from oracle import facodec_oracle as O
    from test_gpu_quantizer_kernels import _sd64, _style_encoder_frames, gamma
    seed = 1
    sd = _sd64(state_dicts(seed)["quantizer"])
    x = _waves(2, 30000, 21)
    t = fb.Codec(_model(seed)).timbre(x).cpu().double()
    with torch.no_grad():
        mel = O.mel_preprocess(sd, x.cpu().double(), n_bins=80)
        mask = torch.ones(mel.size(0), 1, mel.size(2), dtype=torch.bool)
        ref = O.style_encoder(sd, mel, mask)
        y = _style_encoder_frames(sd, mel, mask)
    Tm = mel.size(-1)
    mass = y.abs().amax(1).sum(1) / Tm
    bound = (1e-5 + gamma(Tm // 4 + 2)) * mass[:, None]
    err = (t - ref).abs()
    print("Codec.timbre vs fp64: maxerr %.3e, max err/bound %.3f" % (err.max(), (err / bound).max()))
    assert (err <= bound).all()


def _chunks(total, sizes):
    from test_gpu_stream import chunks_of
    return chunks_of(total, sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("B,sizes", [(1, [3000, 300, 4500, 1200, 9000, 600]), (2, [3300, 6000, 900])])
def test_stream_timbre_every_chunk(B, sizes, built_lib):
    import facodec_b200 as fb
    codec = fb.Codec(_model())
    x = _waves(B, 36000, 60 + B)
    parts = []
    with fb.CodecStream(codec.model, B) as s:
        for p, n in _chunks(x.shape[-1], sizes):
            parts.append(s.encode_codes(x[:, :, p:p + n].contiguous(), 2))
            t = s.timbre()
            assert torch.equal(t, codec.encode(x[:, :, :p + n].contiguous(), 2)[1]), p + n
            assert torch.equal(s.timbre(), t)
        last, timbre = s.finish_codes()
    codes_off, timbre_off = codec.encode(x, 2)
    for i in range(3):
        assert torch.equal(torch.cat([q[i] for q in parts] + [last[i]], dim=2), codes_off[i])
    assert torch.equal(timbre, timbre_off)


@pytest.mark.gpu
def test_stream_timbre_rejections(built_lib):
    import facodec_b200 as fb
    m = _model()
    x = _waves(1, 12000, 3)
    with fb.CodecStream(m, 1) as s:
        with pytest.raises(fb.FacError):
            s.timbre()                                          # before the first chunk
        got = [s.encode_codes(x[:, :, :6000].contiguous(), 2)]
        try:
            m.encoder._engine.set_option("tensor_cores", 1)
            with pytest.raises(fb.FacError):
                s.timbre()
        finally:
            m.encoder._engine.set_option("tensor_cores", 2)
        got.append(s.encode_codes(x[:, :, 6000:].contiguous(), 2))
        last, timbre = s.finish_codes()
        with pytest.raises(fb.FacError):
            s.timbre()                                          # after finish_codes
    codes_off, timbre_off = fb.Codec(m).encode(x, 2)
    for i in range(3):
        assert torch.equal(torch.cat([got[0][i], got[1][i], last[i]], dim=2), codes_off[i])
    assert torch.equal(timbre, timbre_off)
    with fb.CodecStream(m, 1) as s:
        s.encode(x[:, :, :3000].contiguous())
        with pytest.raises(fb.FacError):
            s.timbre()                                          # a latents stream keeps no mel rows


@pytest.mark.gpu
def test_codes_pool_timbre(built_lib):
    """40 sessions, every fifth at 48 kHz, with staggered starts and their own chunk lengths; timbre() over all live ones
    at three points.  Each equals its own B = 1 CodecStream's (for a 48 kHz session: Codec.encode of the 24 kHz frames its
    encoder was fed), the rejected calls change nothing, and every session's codes and final timbre still equal
    Codec.encode of its whole utterance."""
    import facodec_b200 as fb
    codec = fb.Codec(_model())
    rng = random.Random(3)
    S = 40
    rates = [48000 if i % 5 == 4 else 24000 for i in range(S)]
    lens = [rng.choice([30000, 36000, 45000]) for _ in range(S)]
    xs = [_waves(1, int(n * r / 24000), 500 + i) for i, (n, r) in enumerate(zip(lens, rates))]
    joins = [i % 4 for i in range(S)]
    sizes = [[3000 + 300 * rng.randint(0, 20)] + [300 * rng.randint(1, 30) for _ in range(3)] for _ in range(S)]
    pool = fb.CodecStreamPool(codec.model, capacity=S + 4, n_c=2)
    refs = {}                                                   # session -> its B = 1 CodecStream (24 kHz sessions)
    sess, pos, parts, k = {}, [0] * S, {i: [] for i in range(S)}, [0] * S
    fresh = pool.open()                                         # never fed
    short = pool.open(sample_rate=48000)                        # under 3000 samples at 24 kHz
    pool.encode_codes({short: _waves(1, 4000, 9)})
    gone = pool.open()
    pool.close(gone)

    def check_timbres(live):
        got = pool.timbre([sess[i] for i in live])
        assert len(got) == len(live)
        for i in live:
            s = sess[i]
            if rates[i] == 24000:
                ref = refs[i].timbre()
            else:
                fed = pool._fed[s]
                ref = codec.encode(fb.resample(xs[i], 48000, 24000)[..., :fed].contiguous(), 2)[1]
            assert torch.equal(got[s], ref), (i, rates[i])

    step, checks = 0, 0
    while len(sess) < S or any(pos[i] < xs[i].shape[-1] for i in range(S)):
        chunks = {}
        for i in range(S):
            if step < joins[i] or pos[i] >= xs[i].shape[-1]:
                continue
            if i not in sess:
                sess[i] = pool.open(sample_rate=rates[i])
                if rates[i] == 24000:
                    refs[i] = fb.CodecStream(codec.model, 1)
            n = sizes[i][k[i] % len(sizes[i])] if rates[i] == 24000 else rng.choice([1, 2205, 9000, 12000])
            n = min(n, xs[i].shape[-1] - pos[i])
            chunk = xs[i][:, :, pos[i]:pos[i] + n].contiguous()
            chunks[sess[i]] = chunk
            if rates[i] == 24000:
                refs[i].encode_codes(chunk, 2)
            pos[i] += n
            k[i] += 1
        out = pool.encode_codes(chunks)
        for i in range(S):
            if i in sess and sess[i] in out:
                parts[i].append(out[sess[i]])
        live = [i for i in sess if pool._fed[sess[i]] > 0]
        if step in (4, 6, 8) and len(live) > 32:
            check_timbres(live)
            checks += 1
            some = sess[live[0]]
            for bad in ([some, 999], [some, gone], [some, some], [some, fresh], [some, short]):
                with pytest.raises((fb.FacError, ValueError)):
                    pool.timbre(bad)
                # the engine's own checks, behind the wrapper's
                e, out = pool.engine, torch.empty(2, 1024, device="cuda:0")
                rc = e.L.fac_codes_pool_timbre(e.handle, pool.pid, 2, (ctypes.c_int * 2)(*bad),
                                               (ctypes.c_void_p * 2)(out[0].data_ptr(), out[1].data_ptr()), None)
                assert rc < 0, bad
        step += 1
    assert checks >= 2
    fin = pool.finish_codes([sess[i] for i in range(S)])
    with pytest.raises(fb.FacError):
        pool.timbre([sess[0]])                                  # finished
    for i in range(S):
        codes, timbre = fin[sess[i]]
        whole = xs[i] if rates[i] == 24000 else fb.resample(xs[i], 48000, 24000)
        whole = whole[..., :whole.shape[-1] // HOP * HOP].contiguous()
        codes_off, timbre_off = codec.encode(whole, 2)
        got = [torch.cat([p[r] for p in parts[i]] + [codes[r]], dim=2) for r in range(3)]
        for a, b in zip(got, codes_off):
            assert torch.equal(a, b), i
        assert torch.equal(timbre, timbre_off), i
        if i in refs:
            refs[i].close()
    pool.close()


def _codes(T, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 1024, (1, r, T), generator=g).cuda() for r in (1, 2, 3)]


@pytest.mark.gpu
def test_decode_pool_set_timbre(built_lib):
    import facodec_b200 as fb
    m = _model()
    g = torch.Generator().manual_seed(4)
    t0, t1, t2 = (torch.randn(1, 1024, generator=g).cuda() for _ in range(3))
    T = 60
    codes = [_codes(T, 70), _codes(T, 71)]
    pool = fb.CodecDecodePool(m, capacity=4)
    a, b = pool.open(t0), pool.open(t1)
    gone = pool.open(t1)
    pool.close(gone)
    ref = [fb.CodecStream(m, 1), fb.CodecStream(m, 1)]
    voice = [t0, t1]
    outs, refs = [[], []], [[], []]
    cuts = [0, 12, 20, 33, 41, T]
    for j, (p, q) in enumerate(zip(cuts[:-1], cuts[1:])):
        if j == 2:
            pool.set_timbre(a, t2)
            voice[0] = t2
        if j == 3:
            for bad in (t2.view(1024), torch.cat([t2, t2]), t2.cpu()):
                with pytest.raises((ValueError, fb.FacError)):
                    pool.set_timbre(a, bad)
            with pytest.raises(fb.FacError):
                pool.set_timbre(gone, t0)
        chunk = [[c[:, :, p:q] for c in codes[i]] for i in range(2)]
        got = pool.decode_codes({a: chunk[0], b: chunk[1]})
        for i, s in enumerate((a, b)):
            outs[i].append(got[s])
            refs[i].append(ref[i].decode_codes(chunk[i], voice[i]))
    for i in range(2):
        assert torch.equal(torch.cat(outs[i], dim=2), torch.cat(refs[i], dim=2)), i
        ref[i].close()
    pool.finish([b])
    with pytest.raises(fb.FacError):
        pool.set_timbre(b, t0)                                  # ended by finish()
    pool.close()


@pytest.mark.gpu
def test_codec_link_switches_to_sender_voice(built_lib):
    """tx compresses two callers (one at 48 kHz); after 3 s at 24 kHz the receiver switches each session to tx.timbre of
    its caller.  Each receiver's audio equals a B = 1 CodecStream.decode_codes fed the same codes, with the placeholder
    voice before the switch and the sender's after it."""
    import facodec_b200 as fb
    m = _model()
    rates = [24000, 48000]
    xs = [_waves(1, 60000, 90), _waves(1, 120000, 91)]
    placeholder = torch.zeros(1, 1024, device="cuda:0")
    tx = fb.CodecStreamPool(m, capacity=2, n_c=2)
    rx = fb.CodecDecodePool(m, capacity=2)
    ts = [tx.open(sample_rate=r) for r in rates]
    rs = [rx.open(placeholder) for _ in rates]
    refs = [fb.CodecStream(m, 1) for _ in rates]
    voice = [placeholder, placeholder]
    pending = [[], []]
    ys, ys_ref = [[], []], [[], []]
    pos = [0, 0]
    switched = [False, False]

    def deliver(i, codes, final=False):
        pending[i].append(codes)
        frames = sum(q[0].shape[2] for q in pending[i])
        if frames and (ys[i] or final or frames >= 10):
            chunk = [torch.cat([q[r] for q in pending[i]], dim=2) for r in range(3)]
            pending[i].clear()
            ys[i].append(rx.decode_codes({rs[i]: chunk})[rs[i]])
            ys_ref[i].append(refs[i].decode_codes(chunk, voice[i]))

    while any(p < x.shape[-1] for p, x in zip(pos, xs)):
        chunks = {}
        for i, (x, r) in enumerate(zip(xs, rates)):
            if pos[i] < x.shape[-1]:
                n = min(6000 * r // 24000, x.shape[-1] - pos[i])
                chunks[ts[i]] = x[:, :, pos[i]:pos[i] + n]
                pos[i] += n
        out = tx.encode_codes(chunks)
        for i in range(2):
            if ts[i] in out:
                deliver(i, out[ts[i]])
            if not switched[i] and tx._fed[ts[i]] >= 9000:
                t = tx.timbre([ts[i]])[ts[i]]
                rx.set_timbre(rs[i], t)
                voice[i] = t
                switched[i] = True
    fin = tx.finish_codes(ts)
    for i in range(2):
        deliver(i, fin[ts[i]][0], final=True)
        assert switched[i]
        assert torch.equal(torch.cat(ys[i], dim=2), torch.cat(ys_ref[i], dim=2)), rates[i]
        refs[i].close()
    tx.close()
    rx.close()
