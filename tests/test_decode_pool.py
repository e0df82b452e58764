"""The codec decode pool (fac_dec_pool_*; CodecDecodePool): many live receivers decoding codes back to audio in shared
launches, each bit-identical to its own B = 1 CodecStream.decode_codes fed the same chunks and timbre, while the sessions of
one batch differ in chunk length and code rows.  On the host: the launch plan against a restatement.  On the GPU: the
decoder LSTM with per-lane step counts and the per-lane dequantize against B = 1 runs, the pool against B = 1 streams and
Codec.decode, a compression pool chained into a decode pool, and rejected steps leaving every session as it was."""
import ctypes
import math
import random

import numpy as np
import pytest
import torch

from test_stream_pool import plan_engine, plan_restated

DEC_CTX, MIN_FIRST = 20, 10


def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    new = tuple("fac_dec_pool_%s" % c for c in ("create", "open", "decode_codes", "close", "destroy"))
    assert set(new) <= set(_declared("facodec_b200.h"))
    assert "fac_debug_slstm_lanes" in _declared("facodec_b200_debug.h")
    assert set(new) | {"fac_debug_slstm_lanes"} <= set(_lib.EXPORTED)


# ---------------------------------------------------------------------------------------------------------------------
# host: the launch plan
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_decode_pool_plan_matches_restatement(seed, built_lib):
    """The key is the history depth alone: sessions that have decoded equally many frames (any two past 20) share a group
    whatever their chunk lengths; groups over 32 are split."""
    rng = random.Random(seed)
    n = rng.choice([6, 45, 130])
    frames = [0 if rng.random() < 0.15 else rng.choice([10, 12, 19, 20]) if rng.random() < 0.2 else rng.randint(21, 900)
              for _ in range(n)]
    lengths = [rng.randint(MIN_FIRST, 30) if f == 0 else rng.randint(1, 40) for f in frames]
    got = plan_engine(2, frames, lengths)
    assert got == plan_restated([(min(f, DEC_CTX),) for f in frames])
    group, batch, nb = got
    for i in range(n):
        for j in range(n):
            assert (group[i] == group[j]) == (min(frames[i], DEC_CTX) == min(frames[j], DEC_CTX))
    sizes = np.bincount(batch)
    assert sizes.max() <= 32 and len(sizes) == nb
    steady = [lengths[i] for i in range(n) if frames[i] >= DEC_CTX]
    if len(set(steady)) > 1:
        assert len({group[i] for i in range(n) if frames[i] >= DEC_CTX}) == 1     # unequal chunk lengths, one group
    if n == 130:
        assert np.bincount(group).max() > 32 and nb > max(group) + 1


# ---------------------------------------------------------------------------------------------------------------------
# GPU: kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engine(built_lib):
    from facodec_b200.modules import Engine
    e = Engine()
    e._ensure(torch.device("cuda:0"))
    return e


def _lstm_weights(H, seed):
    g = torch.Generator().manual_seed(seed)
    bound = 1.0 / math.sqrt(H)
    return [((torch.rand(s, generator=g) * 2 - 1) * bound).contiguous()
            for _ in range(2) for s in ((4 * H, H), (4 * H, H), (4 * H,), (4 * H,))]


def _slstm_lanes(e, ws, x, lens, carry):
    """fac_debug_slstm_lanes as the decoder's LSTM: x [B][T][H] on the GPU, carry [B][2][words] int32 (updated in place)."""
    B, T, H = x.shape
    arr = (ctypes.c_void_p * 8)(*[w.data_ptr() for w in ws])
    y = torch.full_like(x, float("nan"))
    ln = (ctypes.c_int * B)(*lens) if lens is not None else None
    rc = e.L.fac_debug_slstm_lanes(e.handle, ctypes.c_void_p(x.data_ptr()), arr, B, T, H, 0, ln, ctypes.c_void_p(carry.data_ptr()),
                                   ctypes.c_void_p(y.data_ptr()), None)
    torch.cuda.synchronize()
    assert rc == 0, e.L.fac_last_error(e.handle)
    return y


@pytest.mark.gpu
def test_lstm_lane_lengths_equal_b1_runs(engine):
    """Lane b of a launch with per-lane lengths leaves the (h, c) words a B = 1 launch of lens[b] steps leaves, and writes
    the same output rows up to lens[b]; past them its rows are finite.  Lengths of T everywhere give the bits of no lengths."""
    e = engine
    H = 1536
    words = e.L.fac_debug_lstm_lane_map(H, 0, 0, None, 0)
    ws = _lstm_weights(H, 5)
    g = torch.Generator().manual_seed(9)
    lens = [25, 1, 13, 0, 20, 7, 24]
    B, T = len(lens), 25
    warm = torch.randn(B, 12, H, generator=g).cuda()
    carry0 = torch.zeros(B, 2, words, dtype=torch.int32, device="cuda")
    _slstm_lanes(e, ws, warm, None, carry0)                        # a carried state that is not zero
    assert carry0.abs().sum() > 0
    x = torch.randn(B, T, H, generator=g).cuda()
    carry = carry0.clone()
    y = _slstm_lanes(e, ws, x, lens, carry)
    assert torch.isfinite(y).all()
    for b, n in enumerate(lens):
        if n == 0:
            assert torch.equal(carry[b], carry0[b])
            continue
        c1 = carry0[b:b + 1].clone()
        y1 = _slstm_lanes(e, ws, x[b:b + 1, :n].contiguous(), None, c1)
        assert torch.equal(carry[b], c1[0]), b
        assert torch.equal(y[b, :n], y1[0]), b
    c_full, c_none = carry0.clone(), carry0.clone()
    y_full = _slstm_lanes(e, ws, x, [T] * B, c_full)
    y_none = _slstm_lanes(e, ws, x, None, c_none)
    assert torch.equal(c_full, c_none) and torch.equal(y_full, y_none)


def _model():
    from test_gpu_parity import model_for
    return model_for(0)


def _random_codes(T, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 1024, (1, r, T), generator=g).cuda() for r in (1, 2, 3)]


def _chunk(codes, p, F, nc, nr):
    cp, cc, cr = codes
    return [cp[:, :, p:p + F], cc[:, :nc, p:p + F], cr[:, :nr, p:p + F] if nr else None]


@pytest.mark.gpu
def test_dequantize_lanes_equal_dequantize(built_lib):
    """The pool's per-lane dequantize (tapped as dec_pool.latents) against FAquantizer.from_codes of each lane's own codes,
    rows and timbre: valid frames bit-identical, padding frames zero."""
    import facodec_b200 as fb
    m = _model()
    e = m.decoder._engine
    spec = [(12, 1, 0), (10, 2, 3), (17, 2, 1), (11, 1, 2)]
    Fmax = max(s[0] for s in spec)
    tvs = [torch.randn(1, 1024, generator=torch.Generator().manual_seed(60 + i)).cuda() for i in range(len(spec))]
    codes = [_random_codes(F, 70 + i) for i, (F, _, _) in enumerate(spec)]
    buf = torch.full((len(spec), Fmax, 1024), float("nan"), device="cuda")
    with fb.CodecDecodePool(m, capacity=len(spec)) as pool:
        sid = [pool.open(tv) for tv in tvs]
        e.L.fac_debug_tap(e.handle, b"dec_pool.latents", ctypes.c_void_p(buf.data_ptr()), buf.numel())
        try:
            pool.decode_codes({sid[i]: _chunk(codes[i], 0, F, nc, nr) for i, (F, nc, nr) in enumerate(spec)})
            torch.cuda.synchronize()
        finally:
            e.L.fac_debug_tap(e.handle, b"dec_pool.latents", None, 0)
    for b, (F, nc, nr) in enumerate(spec):
        ref, _ = m.quantizer.from_codes(_chunk(codes[b], 0, F, nc, nr), tvs[b])
        assert torch.equal(buf[b, :F], ref[0].transpose(0, 1)), b
        assert torch.equal(buf[b, F:], torch.zeros_like(buf[b, F:])), b


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the pool
# ---------------------------------------------------------------------------------------------------------------------
def _dec_schedule(rng, n, late=4, vary_rows=True):
    """n receivers starting over the first 3 steps with 15-25-frame chunks (a first chunk of 10-25; a few take a 1- and a
    40-frame chunk), code rows switching between steps when vary_rows; sessions 2, 9, 14, 21 leave after two chunks, and
    `late` more open at step 8 into the freed slots."""
    out = []
    for i in range(n + late):
        steps = rng.randint(4, 9)
        Fs = [rng.randint(MIN_FIRST, 25)] + [rng.randint(15, 25) for _ in range(steps - 1)]
        if i % 7 == 3:
            Fs[1:3] = [1, 40]
        fixed = (rng.choice([1, 2]), rng.choice([0, 1, 2, 3]))
        rows = [(rng.choice([1, 2]), rng.choice([0, 1, 2, 3])) if vary_rows else fixed for _ in Fs]
        abandon = i in (2, 9, 14, 21)
        out.append(dict(codes=_random_codes(sum(Fs), 5000 + i),
                        tv=torch.randn(1, 1024, generator=torch.Generator().manual_seed(6000 + i)).cuda(),
                        Fs=Fs[:2] if abandon else Fs, rows=rows, start=8 if i >= n else rng.randint(0, 2)))
    return out


def _chunks(s):
    p = 0
    for F, (nc, nr) in zip(s["Fs"], s["rows"]):
        yield _chunk(s["codes"], p, F, nc, nr)
        p += F


def _run_dec_pool(pool, sched):
    """Steps the pool through the schedule; returns per session its output chunks, and per step the plan's batches as
    lists of (F, rows) of their members."""
    res = [[] for _ in sched]
    feeds = [list(_chunks(s)) for s in sched]
    sid, done, step, frames, batches = {}, set(), 0, [0] * len(sched), []
    while len(done) < len(sched):
        for i, s in enumerate(sched):
            if s["start"] == step:
                sid[i] = pool.open(s["tv"])
        feed = {i: feeds[i][len(res[i])] for i in sid if i not in done and len(res[i]) < len(feeds[i])}
        if feed:
            order = list(feed)
            _, batch, nb = plan_engine(2, [frames[i] for i in order], [feed[i][0].shape[2] for i in order])
            batches.append([[(feed[i][0].shape[2], feed[i][1].shape[1], 0 if feed[i][2] is None else feed[i][2].shape[1])
                             for k, i in enumerate(order) if batch[k] == j] for j in range(nb)])
        out = pool.decode_codes({sid[i]: c for i, c in feed.items()})
        for i, c in feed.items():
            res[i].append(out[sid[i]])
            frames[i] += c[0].shape[2]
            if len(res[i]) == len(feeds[i]):
                pool.close(sid[i])
                done.add(i)
        step += 1
    return res, batches


def _b1(m, s):
    import facodec_b200 as fb
    with fb.CodecStream(m, 1) as st:
        return [st.decode_codes(c, s["tv"]) for c in _chunks(s)]


@pytest.mark.gpu
def test_decode_pool_equals_b1_streams(built_lib):
    import facodec_b200 as fb
    m = _model()
    sched = _dec_schedule(random.Random(21), 40)
    with fb.CodecDecodePool(m, capacity=40) as pool:
        res, batches = _run_dec_pool(pool, sched)
        with pytest.raises(fb.FacError):
            for _ in range(41):
                pool.open(sched[0]["tv"])                               # past capacity
    flat = [b for step in batches for b in step]
    assert max(len(b) for b in flat) == 32 and max(len(step) for step in batches) > 2   # a group over 32 was split
    assert any(len({f for f, _, _ in b}) > 1 for b in flat)                            # batches mix chunk lengths,
    assert any(len({nc for _, nc, _ in b}) > 1 and len({nr for _, _, nr in b}) > 2 for b in flat)   # and code rows
    for i, s in enumerate(sched):
        ref = _b1(m, s)
        assert len(ref) == len(res[i])
        for k, (a, b) in enumerate(zip(res[i], ref)):
            assert torch.equal(a, b), (i, k)


@pytest.mark.gpu
def test_decode_pool_equals_offline_decode(built_lib):
    """Concatenated pool output against Codec.decode on the whole code sequence, at the bar of the stream's own test."""
    import facodec_b200 as fb
    m = _model()
    sched = _dec_schedule(random.Random(5), 8, late=0, vary_rows=False)
    with fb.CodecDecodePool(m, capacity=8) as pool:
        res, batches = _run_dec_pool(pool, sched)
    assert any(len({f for f, _, _ in b}) > 1 for step in batches for b in step)
    for i, s in enumerate(sched):
        nc, nr = s["rows"][0]
        T = sum(s["Fs"])
        y_off = fb.Codec(m).decode(_chunk(s["codes"], 0, T, nc, nr), s["tv"])
        y = torch.cat(res[i], dim=2)
        assert y.shape == y_off.shape
        assert float(((y.double() - y_off.double()) ** 2).mean().sqrt()) <= 1e-4, i


@pytest.mark.gpu
def test_codes_pool_into_decode_pool_equals_stream_pair(built_lib):
    """A codec link for 12 callers: the compression pool's codes go straight into the decode pool (a 19-frame first chunk,
    20-frame chunks, the 1-frame finish), bit-identical to one CodecStream per caller doing encode_codes -> decode_codes."""
    import facodec_b200 as fb
    from test_gpu_stream import chunks_of
    from facodec_b200 import synth
    m = _model()
    rng = random.Random(13)
    n = 12
    xs = [synth.synth_waves(1, 300 * rng.randint(60, 150), seed=7000 + i).to("cuda:0") for i in range(n)]
    tvs = [torch.randn(1, 1024, generator=torch.Generator().manual_seed(7100 + i)).cuda() for i in range(n)]
    starts = [rng.randint(0, 2) for _ in range(n)]
    chunks = [chunks_of(x.shape[-1], [6000]) for x in xs]
    ys = [[] for _ in range(n)]
    with fb.CodecStreamPool(m, capacity=n, n_c=2) as tx, fb.CodecDecodePool(m, capacity=n) as rx:
        cs, rs, k, step = {}, {}, [0] * n, 0
        while any(k[i] < len(chunks[i]) for i in range(n)):
            for i in range(n):
                if starts[i] == step:
                    cs[i], rs[i] = tx.open(), rx.open(tvs[i])
            feed = {i: xs[i][:, :, p:p + q].contiguous() for i in cs if k[i] < len(chunks[i]) for p, q in [chunks[i][k[i]]]}
            codes = tx.encode_codes({cs[i]: x for i, x in feed.items()})
            ending = [i for i in feed if k[i] + 1 == len(chunks[i])]
            fin = tx.finish_codes([cs[i] for i in ending])
            out = rx.decode_codes({rs[i]: codes[cs[i]] for i in feed})
            for i in feed:
                ys[i].append(out[rs[i]])
                k[i] += 1
            if ending:
                out = rx.decode_codes({rs[i]: fin[cs[i]][0] for i in ending})
                for i in ending:
                    ys[i].append(out[rs[i]])
                    tx.close(cs[i])
                    rx.close(rs[i])
            step += 1
    for i in range(n):
        with fb.CodecStream(m, 1) as st:
            ref = [st.decode_codes(st.encode_codes(xs[i][:, :, p:p + q].contiguous(), 2), tvs[i]) for p, q in chunks[i]]
            ref.append(st.decode_codes(st.finish_codes()[0], tvs[i]))
        assert len(ref) == len(ys[i]) and all(torch.equal(a, b) for a, b in zip(ys[i], ref)), i


@pytest.mark.gpu
def test_rejected_steps_leave_sessions_unchanged(built_lib):
    import facodec_b200 as fb
    from facodec_b200.modules import _ptr_array, _stream
    m = _model()
    e = m.decoder._engine
    specs = [dict(codes=_random_codes(60, 90 + i), tv=torch.randn(1, 1024, generator=torch.Generator().manual_seed(95 + i)).cuda(),
                  Fs=Fs, rows=rows) for i, (Fs, rows) in enumerate((([12, 20, 28], [(2, 3), (1, 0), (2, 2)]),
                                                                     ([10, 25, 25], [(1, 0), (2, 3), (1, 1)])))]
    parts = [list(_chunks(s)) for s in specs]
    with fb.CodecDecodePool(m, capacity=4) as pool:
        a, b = pool.open(specs[0]["tv"]), pool.open(specs[1]["tv"])
        got = {a: [], b: []}
        for s, y in pool.decode_codes({a: parts[0][0], b: parts[1][0]}).items():
            got[s].append(y)
        fresh, closed = pool.open(specs[0]["tv"]), pool.open(specs[0]["tv"])
        pool.close(closed)
        good = {a: parts[0][1], b: parts[1][1]}
        cp, cc, cr = _random_codes(12, 99)
        bad_codes = cr.clone()
        bad_codes[0, 1, 4] = 1024
        for bad, err in (({**good, fresh: [c[:, :, :9] for c in (cp, cc, cr)]}, fb.FacError),  # a first chunk under 10 frames
                         ({**good, fresh: [cp, cc.repeat(1, 2, 1), cr]}, ValueError),        # 4 content rows
                         ({**good, fresh: [cp, cc, bad_codes]}, IndexError),                  # an out-of-range code
                         ({**good, fresh: [cp.cpu(), cc.cpu(), cr.cpu()]}, fb.FacError),     # a CPU tensor
                         ({**good, closed: [cp, cc, cr]}, fb.FacError)):                      # a session not open
            with pytest.raises(err):
                pool.decode_codes(bad)
        # through the C entry point: rows outside the bounds the Python layer enforces, and a session named twice
        P = lambda ts: _ptr_array(ctypes.c_void_p, [t.data_ptr() for t in ts])
        ys = [torch.empty(300 * 12, device="cuda") for _ in range(2)]
        I = lambda v: _ptr_array(ctypes.c_int, v)
        for sess, nc, nr in (([a, fresh], [1, 3], [0, 0]), ([a, fresh], [1, 1], [0, 4]), ([a, fresh], [0, 1], [0, 0]),
                             ([a, a], [1, 1], [0, 0])):
            rc = e.L.fac_dec_pool_decode_codes(e.handle, pool.pid, 2, I(sess), I([12, 12]), P([cp, cp]), P([cc, cc]), I(nc),
                                               P([cr, cr]), I(nr), P(ys), _stream(cp.device))
            assert rc == -1
        for step in (1, 2):
            for s, y in pool.decode_codes({a: parts[0][step], b: parts[1][step]}).items():
                got[s].append(y)
    for s, spec in ((a, specs[0]), (b, specs[1])):
        ref = _b1(m, spec)
        assert len(ref) == len(got[s]) and all(torch.equal(x, y) for x, y in zip(got[s], ref)), s
