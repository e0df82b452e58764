"""Stream pools (fac_codes_pool_*, fac_vc_pool_*; CodecStreamPool, VoiceConversionPool): many live sessions stepped in shared
launches, each bit-identical to its own B = 1 stream fed the same chunks, whatever the interleaving of opens, steps, finishes
and closes.  On the host: the launch plan against a restatement of the grouping, and the LSTM carry's lane map.  On the GPU:
the pools against B = 1 streams and the offline calls, and rejected steps leaving every session as it was."""
import ctypes
import random

import numpy as np
import pytest
import torch

HOP, WN_CTX, ENC_CTX, RED_CTX, DEC_CTX = 300, 32, 6000, 32, 12


def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    new = tuple("fac_%s_pool_%s" % (k, c) for k in ("codes", "vc") for c in ("create", "open", "close", "destroy")) + (
        "fac_codes_pool_encode_codes", "fac_codes_pool_finish_codes", "fac_vc_pool_convert", "fac_vc_pool_finish")
    assert set(new) <= set(_declared("facodec_b200.h"))
    assert {"fac_debug_pool_plan", "fac_debug_lstm_lane_map"} <= set(_declared("facodec_b200_debug.h"))
    assert set(new) | {"fac_debug_pool_plan", "fac_debug_lstm_lane_map"} <= set(_lib.EXPORTED)


# ---------------------------------------------------------------------------------------------------------------------
# host: the launch plan
# ---------------------------------------------------------------------------------------------------------------------
def codes_counters(enc_samples):
    """A B = 1 compression stream's counters after enc_samples samples: (enc_samples, x_hist_len, ey_hist_len, emitted)."""
    return (enc_samples, min(enc_samples, ENC_CTX), min(enc_samples // HOP, 2), max(enc_samples // HOP - 1, 0))


def codes_key(c, T):
    enc, hist, yh, E = c
    N = (enc + T) // HOP
    Fout, lo = N - 1 - E, max(E - WN_CTX, 0)
    return (T, hist, yh, enc == 0, E - (enc - hist) // HOP, Fout, E - lo, E + Fout - lo)


def vc_counters(N):
    """A B = 1 voice-conversion stream's (N, Zf, Yf) after N code frames."""
    Zf = max(N - RED_CTX, 0)
    return (N, Zf, max(Zf - DEC_CTX, 0))


def vc_key(c, F):
    N, Zf, Yf = c
    Zf1 = max(N + F - RED_CTX, Zf)
    Yf1 = max(Zf1 - DEC_CTX, Yf)
    hc0, zh0, hc1, zh1 = max(Zf - RED_CTX, 0), max(Yf - DEC_CTX, 0), max(Zf1 - RED_CTX, 0), max(Yf1 - DEC_CTX, 0)
    return (F, N + F - hc0, N - hc0, Zf1 - zh0, Zf - zh0, Zf1 - Zf, Yf1 - Yf, Yf - zh0, zh1 - zh0, Zf1 - zh1, hc1 - hc0,
            N + F - hc1)


def plan_restated(keys):
    """Groups in order of first appearance, members in input order, batches of <= 32."""
    order, members = [], {}
    for i, k in enumerate(keys):
        if k not in members:
            order.append(k)
            members[k] = []
        members[k].append(i)
    group, batch, nb = [0] * len(keys), [0] * len(keys), 0
    for g, k in enumerate(order):
        m = members[k]
        for o in range(0, len(m), 32):
            for i in m[o:o + 32]:
                group[i], batch[i] = g, nb
            nb += 1
    return group, batch, nb


def plan_engine(kind, counters, lengths):
    from facodec_b200 import _lib
    L = _lib.load()
    n = len(lengths)
    c = np.ascontiguousarray(np.array(counters, dtype=np.int64).reshape(-1))
    ln = np.array(lengths, dtype=np.int32)
    group, batch = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    nb = L.fac_debug_pool_plan(kind, n, P(c), P(ln), P(group), P(batch))
    assert nb >= 0
    return list(group), list(batch), nb


@pytest.mark.parametrize("seed", range(6))
def test_codes_pool_plan_matches_restatement(seed, built_lib):
    rng = random.Random(seed)
    n = rng.choice([5, 40, 120])
    counters, lengths = [], []
    for _ in range(n):
        steady = rng.random() < 0.7
        enc = 300 * rng.randint(40, 400) if steady else rng.choice([0, 3000, 6000, 6300, 9000])
        counters.append(codes_counters(enc))
        lengths.append(rng.choice([6000] * 10 + [300, 3000, 3900, 15000]))
    keys = [codes_key(c, T) for c, T in zip(counters, lengths)]
    got = plan_engine(0, counters, lengths)
    assert got == plan_restated(keys)
    group, batch, nb = got
    # steady-state sessions (prosody window full) with equal chunk lengths share one group; warm-up ones do not join it
    for i in range(n):
        for j in range(n):
            si, sj = counters[i][3] > WN_CTX + 1, counters[j][3] > WN_CTX + 1
            if si and sj and lengths[i] == lengths[j]:
                assert group[i] == group[j]
            if si != sj:
                assert group[i] != group[j]
    sizes = np.bincount(batch)
    assert sizes.max() <= 32 and len(sizes) == nb
    if n == 120:
        assert np.bincount(group).max() > 32 and nb > max(group) + 1      # a group larger than 32 was split


@pytest.mark.parametrize("seed", range(6))
def test_vc_pool_plan_matches_restatement(seed, built_lib):
    rng = random.Random(100 + seed)
    n = rng.choice([7, 50, 70])
    counters = [vc_counters(rng.choice([0, 1, 20, 40, 44, 60]) if rng.random() < 0.3 else rng.randint(70, 900)) for _ in range(n)]
    lengths = [rng.choice([20] * 5 + [1, 7, 13, 50]) for _ in range(n)]
    keys = [vc_key(c, F) for c, F in zip(counters, lengths)]
    got = plan_engine(1, counters, lengths)
    assert got == plan_restated(keys)
    group, batch, _ = got
    for i in range(n):
        for j in range(n):
            if counters[i][0] >= 64 and counters[j][0] >= 64 and lengths[i] == lengths[j]:
                assert group[i] == group[j]
            if lengths[i] != lengths[j] or (counters[i][0] < 64) != (counters[j][0] < 64):
                assert group[i] != group[j]
    assert np.bincount(batch).max() <= 32


# ---------------------------------------------------------------------------------------------------------------------
# host: the LSTM carry's lane map
# ---------------------------------------------------------------------------------------------------------------------
def lane_map(H, pass3, lane):
    from facodec_b200 import _lib
    L = _lib.load()
    n = L.fac_debug_lstm_lane_map(H, pass3, lane, None, 0)
    assert n == (2 if pass3 else 1) * H // 2 + H
    pos = np.zeros(n, dtype=np.int64)
    assert L.fac_debug_lstm_lane_map(H, pass3, lane, pos.ctypes.data_as(ctypes.c_void_p), n) == n
    return pos


@pytest.mark.parametrize("H", [1024, 1536])
@pytest.mark.parametrize("pass3", [0, 1])
def test_lstm_lane_map_is_a_bijection(H, pass3, built_lib):
    """Lane b's carry words are exactly the state words the recurrence kernel reads and writes for batch column b: h word
    (plane, k pair kp) of lane b at plane * H/2 * 32 + kp * 32 + (b ^ ((kp & 3) << 3)), c of unit k at the CTA's [32][U]
    tile.  Over the 32 lanes the maps partition the state, and moving lane b into lane b' and back is the identity."""
    PL = 2 if pass3 else 1
    U = 8 if H == 1024 else 12
    hw = PL * (H // 2) * 32
    total = hw + H * 32
    maps = [lane_map(H, pass3, b) for b in range(32)]
    allpos = np.concatenate(maps)
    assert np.array_equal(np.sort(allpos), np.arange(total))
    for b, m in enumerate(maps):
        h, c = m[:PL * H // 2], m[PL * H // 2:]
        kp = np.arange(PL * H // 2) % (H // 2)
        assert np.all(h < hw) and np.all(c >= hw)
        assert np.array_equal(h % 32, b ^ ((kp & 3) << 3))
        k = np.arange(H)
        assert np.array_equal(c - hw, (k // U) * 32 * U + b * U + k % U)
    rng = np.random.default_rng(H + pass3)
    state = rng.integers(0, 2 ** 32, total, dtype=np.uint64).astype(np.uint32)
    for b, b2 in ((0, 31), (5, 9), (17, 17)):
        moved = state.copy()
        moved[maps[b2]] = state[maps[b]]              # lane b -> lane b'
        back = moved.copy()
        back[maps[b]] = moved[maps[b2]]               # and back
        assert np.array_equal(back[maps[b]], state[maps[b]])
        assert np.array_equal(moved[maps[b2]], state[maps[b]])


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
MIXED_CHUNKINGS = [[3000, 300, 15000, 3900], [3000], [3900, 300], [3000, 300, 15000, 3900]]


def _wave(T, seed):
    from facodec_b200 import synth
    return synth.synth_waves(1, T, seed=seed).to("cuda:0")


def _codec_schedule(rng, n, late=4):
    """n sessions of 1.5-6 s starting over the first 3 steps, all but 4 in 0.25 s chunks (so at step 4 more than 32 of them
    share one launch sequence); sessions 3, 7, 11, 19 are closed after five chunks, and `late` more sessions open at step 8
    into the freed slots."""
    from test_gpu_stream import chunks_of
    out = []
    for i in range(n + late):
        T = 300 * rng.randint(120, 480)
        chunks = chunks_of(T, MIXED_CHUNKINGS[i // 9] if i in (0, 9, 18, 27) else [6000])
        abandon = i in (3, 7, 11, 19)
        out.append(dict(x=_wave(T, 1000 + i), start=8 if i >= n else rng.randint(0, 2),
                        chunks=chunks[:5] if abandon else chunks, finish=not abandon))
    return out


def _run_codec_pool(pool, sched, on_step=None):
    """Steps the pool through the schedule; returns per session (codes chunks, finish result or None) and the largest group
    a step held (by the restated keys)."""
    res = [dict(codes=[], fin=None) for _ in sched]
    sid, done, step, biggest = {}, set(), 0, 0
    while len(done) < len(sched):
        for i, s in enumerate(sched):
            if s["start"] == step:
                sid[i] = pool.open()
        feed, keys = {}, []
        for i, s in enumerate(sched):
            k = len(res[i]["codes"])
            if i in sid and i not in done and k < len(s["chunks"]):
                p, n = s["chunks"][k]
                feed[i] = s["x"][:, :, p:p + n].contiguous()
                keys.append(codes_key(codes_counters(p), n))
        if keys:
            biggest = max(biggest, max(keys.count(k) for k in keys))
        out = pool.encode_codes({sid[i]: x for i, x in feed.items()})
        for i in feed:
            res[i]["codes"].append(out[sid[i]])
            if on_step:
                on_step(i, out[sid[i]])
        ending = [i for i in feed if len(res[i]["codes"]) == len(sched[i]["chunks"])]
        fin = pool.finish_codes([sid[i] for i in ending if sched[i]["finish"]])
        for i in ending:
            if sched[i]["finish"]:
                res[i]["fin"] = fin[sid[i]]
            pool.close(sid[i])
            done.add(i)
        step += 1
    return res, biggest


def _codec_b1(codec, s):
    import facodec_b200 as fb
    with fb.CodecStream(codec, 1) as tx:
        codes = [tx.encode_codes(s["x"][:, :, p:p + n].contiguous(), 2) for p, n in s["chunks"]]
        fin = tx.finish_codes() if s["finish"] else None
    return codes, fin


def _cat_codes(chunks, last=None):
    return [torch.cat([c[i] for c in chunks] + ([last[i]] if last is not None else []), dim=2) for i in range(3)]


@pytest.mark.gpu
def test_codes_pool_equals_b1_streams(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import model_for
    codec = model_for(0)
    sched = _codec_schedule(random.Random(7), 40)
    with fb.CodecStreamPool(codec, capacity=40, n_c=2) as pool:
        res, biggest = _run_codec_pool(pool, sched)
        with pytest.raises(fb.FacError):
            for _ in range(41):
                pool.open()                                  # past capacity
    assert biggest > 32
    for i, s in enumerate(sched):
        codes, fin = _codec_b1(codec, s)
        for a, b in zip(res[i]["codes"], codes):
            assert all(torch.equal(x, y) for x, y in zip(a, b)), i
        if s["finish"]:
            assert all(torch.equal(x, y) for x, y in zip(res[i]["fin"][0], fin[0])), i
            assert torch.equal(res[i]["fin"][1], fin[1]), i
            codes_off, timbre_off = fb.Codec(codec).encode(s["x"], 2)
            got = _cat_codes(res[i]["codes"], res[i]["fin"][0])
            assert all(torch.equal(x, y) for x, y in zip(got, codes_off)), i
            assert torch.equal(res[i]["fin"][1], timbre_off), i


def _vc_schedule(rng, n, late=4):
    from test_gpu_stream import chunks_of
    out = []
    for i in range(n + late):
        T = rng.randint(60, 240)
        g = torch.Generator().manual_seed(2000 + i)
        cp, cc = torch.randint(0, 1024, (1, 1, T), generator=g), torch.randint(0, 1024, (1, 2, T), generator=g)
        tv = torch.randn(1, 1024, generator=g)
        chunks = chunks_of(T, rng.choice([[20]] * 5 + [[7, 1, 50, 13], [1], [13]]))
        abandon = i in (2, 9, 14, 21)
        out.append(dict(cp=cp.cuda(), cc=cc.cuda(), tv=tv.cuda(), start=8 if i >= n else rng.randint(0, 3),
                        chunks=chunks[:2] if abandon else chunks, finish=not abandon))
    return out


def _run_vc_pool(pool, sched):
    res = [[] for _ in sched]
    sid, done, step, fed = {}, set(), 0, [0] * len(sched)
    while len(done) < len(sched):
        for i, s in enumerate(sched):
            if s["start"] == step:
                sid[i] = pool.open(s["tv"])
        feed = {}
        for i, s in enumerate(sched):
            if i in sid and i not in done and fed[i] < len(s["chunks"]):
                p, n = s["chunks"][fed[i]]
                feed[i] = [s["cp"][:, :, p:p + n], s["cc"][:, :, p:p + n]]
                fed[i] += 1
        out = pool.convert({sid[i]: c for i, c in feed.items()})
        for i in feed:
            res[i].append(out[sid[i]])
        ending = [i for i in feed if fed[i] == len(sched[i]["chunks"])]
        fin = pool.finish([sid[i] for i in ending if sched[i]["finish"]])
        for i in ending:
            if sched[i]["finish"]:
                res[i].append(fin[sid[i]])
            pool.close(sid[i])
            done.add(i)
        step += 1
    return res


@pytest.mark.gpu
def test_vc_pool_equals_b1_streams(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    sched = _vc_schedule(random.Random(3), 40)
    with fb.VoiceConversionPool(m, capacity=40, use_p_code=False, use_c_code=True, n_c=1) as pool:
        res = _run_vc_pool(pool, sched)
    for i, s in enumerate(sched):
        with fb.VoiceConversionStream(m, 1, s["tv"], use_p_code=False, n_c=1) as vs:
            ref = [vs.convert([s["cp"][:, :, p:p + n], s["cc"][:, :, p:p + n]]) for p, n in s["chunks"]]
            if s["finish"]:
                ref.append(vs.finish())
        assert len(ref) == len(res[i]) and all(torch.equal(a, b) for a, b in zip(res[i], ref)), i
        if s["finish"]:
            y_off = fb.VoiceConverter(m).convert([s["cp"], s["cc"]], s["tv"], use_p_code=False, n_c=1)
            assert torch.equal(torch.cat(res[i], dim=2), y_off), i


@pytest.mark.gpu
def test_chained_pools_equal_offline(built_lib):
    """Live voice conversion for 34 callers: the codec pool's codes go straight into the voice-conversion pool."""
    import facodec_b200 as fb
    from test_gpu_parity import model_for, redec_model_for
    from test_gpu_stream import chunks_of
    codec, rm = model_for(0), redec_model_for(0)
    rng = random.Random(11)
    n = 34
    xs = [_wave(300 * rng.randint(120, 240), 3000 + i) for i in range(n)]
    targets = [torch.randn(1, 1024, generator=torch.Generator().manual_seed(i)).cuda() for i in range(n)]
    starts = [rng.randint(0, 2) for _ in range(n)]
    chunks = [chunks_of(x.shape[-1], [6000]) for x in xs]
    ys = [[] for _ in range(n)]
    with fb.CodecStreamPool(codec, capacity=n, n_c=2) as tx, fb.VoiceConversionPool(rm, capacity=n, n_c=1) as vc:
        cs, vs, k, step = {}, {}, [0] * n, 0
        while any(k[i] <= len(chunks[i]) for i in range(n)):
            for i in range(n):
                if starts[i] == step:
                    cs[i], vs[i] = tx.open(), vc.open(targets[i])
            feed = {i: xs[i][:, :, p:p + m].contiguous() for i in cs if k[i] < len(chunks[i])
                    for p, m in [chunks[i][k[i]]]}
            codes = tx.encode_codes({cs[i]: x for i, x in feed.items()})
            ending = [i for i in feed if k[i] + 1 == len(chunks[i])]
            fin = tx.finish_codes([cs[i] for i in ending])
            conv = {vs[i]: codes[cs[i]] for i in feed}
            out = vc.convert(conv)
            for i in feed:
                ys[i].append(out[vs[i]])
                k[i] += 1
            if ending:
                out = vc.convert({vs[i]: fin[cs[i]][0] for i in ending})
                tail = vc.finish([vs[i] for i in ending])
                for i in ending:
                    ys[i] += [out[vs[i]], tail[vs[i]]]
                    tx.close(cs[i])
                    vc.close(vs[i])
                    k[i] += 1
            step += 1
    for i in range(n):
        codes_off, _ = fb.Codec(codec).encode(xs[i], 2)
        y_off = fb.VoiceConverter(rm).convert(codes_off, targets[i], use_p_code=False, n_c=1)
        assert torch.equal(torch.cat(ys[i], dim=2), y_off), i


@pytest.mark.gpu
def test_rejected_steps_leave_sessions_unchanged(built_lib):
    import facodec_b200 as fb
    from facodec_b200.modules import _ptr_array, _stream
    from test_gpu_parity import model_for, redec_model_for
    codec, rm = model_for(0), redec_model_for(0)
    xa, xb = _wave(18000, 51), _wave(18000, 52)
    with fb.CodecStreamPool(codec, capacity=4, n_c=2) as pool:
        a, b = pool.open(), pool.open()
        got = {a: [], b: []}
        for s, v in pool.encode_codes({a: xa[:, :, :6000], b: xb[:, :, :3000]}).items():
            got[s].append(v)
        fresh, closed = pool.open(), pool.open()
        pool.close(closed)
        good = {a: xa[:, :, 6000:12000], b: xb[:, :, 3000:6000]}
        for bad in ({**good, closed: xa[:, :, :6000]},                 # a closed session
                    {**good, fresh: xa[:, :, :2700]},                  # a first chunk under 3000 samples
                    {**good, fresh: xa[:, :, :3100]},                  # T not a multiple of 300
                    {a: xa[:, :, 6000:12000], b: xb[:, :, 3000:3150]}):
            with pytest.raises((fb.FacError, ValueError)):
                pool.encode_codes(bad)
        # a duplicate session, through the C entry point (a dict cannot name one twice)
        e = codec.encoder._engine
        x1 = xa[:, :, 6000:12000].contiguous()
        outs = [torch.empty(1, r, 20, dtype=torch.int64, device="cuda:0") for r in (1, 2, 3)] * 2
        P = lambda ts: _ptr_array(ctypes.c_void_p, [t.data_ptr() for t in ts])
        frames = (ctypes.c_int * 2)()
        rc = e.L.fac_codes_pool_encode_codes(e.handle, pool.pid, 2, _ptr_array(ctypes.c_int, [a, a]), _ptr_array(ctypes.c_int, [6000, 6000]),
                                             P([x1, x1]), P(outs[0::3]), P(outs[1::3]), P(outs[2::3]), frames, _stream(x1.device))
        assert rc == -1
        for s, v in pool.encode_codes(good).items():
            got[s].append(v)
        for s, v in pool.encode_codes({a: xa[:, :, 12000:], b: xb[:, :, 6000:]}).items():
            got[s].append(v)
        fin = pool.finish_codes([a, b])
    for s, x in ((a, xa), (b, xb)):
        codes_off, timbre_off = fb.Codec(codec).encode(x, 2)
        assert all(torch.equal(p, q) for p, q in zip(_cat_codes(got[s], fin[s][0]), codes_off))
        assert torch.equal(fin[s][1], timbre_off)

    g = torch.Generator().manual_seed(5)
    cp, cc, tv = (torch.randint(0, 1024, (2, 1, 80), generator=g).cuda(), torch.randint(0, 1024, (2, 2, 80), generator=g).cuda(),
                  torch.randn(2, 1024, generator=g).cuda())
    with fb.VoiceConversionPool(rm, capacity=2, n_c=1) as vp:
        v = [vp.open(tv[i:i + 1]) for i in range(2)]
        with pytest.raises(fb.FacError):
            vp.open(tv[:1])                                             # full
        ys = [[], []]
        part = lambda i, lo, hi: [cp[i:i + 1, :, lo:hi], cc[i:i + 1, :, lo:hi]]
        for i, y in enumerate(vp.convert({v[0]: part(0, 0, 40), v[1]: part(1, 0, 40)}).values()):
            ys[i].append(y)
        bad = cc[1:2, :, 40:80].clone()
        bad[0, 0, 3] = 1024
        with pytest.raises(IndexError):
            vp.convert({v[0]: part(0, 40, 80), v[1]: [cp[1:2, :, 40:80], bad]})
        with pytest.raises(fb.FacError):
            vp.finish([v[0], 7])                                        # unknown session
        out = vp.convert({v[0]: part(0, 40, 80), v[1]: part(1, 40, 80)})
        tail = vp.finish(v)
        vp.close(v[1])
        with pytest.raises(fb.FacError):
            vp.convert({v[1]: part(1, 0, 5)})                           # closed
    for i in range(2):
        y = torch.cat(ys[i] + [out[v[i]], tail[v[i]]], dim=2)
        assert torch.equal(y, fb.VoiceConverter(rm).convert([cp[i:i + 1], cc[i:i + 1]], tv[i:i + 1], use_p_code=False, n_c=1))
