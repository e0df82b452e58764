"""Switching a live voice conversion's target voice mid-stream, and mixing conversion modes in one voice-conversion pool
(fac_vc_stream_set_timbre, fac_vc_pool_set_timbre, fac_vc_pool_open_mode; VoiceConversionStream.set_timbre,
VoiceConversionPool.set_timbre / open(..., use_p_code, use_c_code, n_c)).

After a switch before call k, every sample that call k, the later calls and finish emit equals VoiceConverter.convert of the
whole utterance with the new timbre at the same positions, and what was emitted before equals it with the old timbre: the
output is a splice of offline conversions at the output frame Yf of each switch.  The step after a switch recomputes the z
frames [Yf - 12, Zf) the decoder still reads from codes back to Yf - 12 - 32, so the stream keeps the last 2 * (32 + 12) code
frames.  On the host: that plan against a restatement, and the history bound along random walks.  On the GPU: the splices
bit for bit, mixed modes in one launch sequence, switches inside a pool and at 48 kHz, and rejected calls."""
import ctypes
import random

import numpy as np
import pytest
import torch

RED_CTX, DEC_CTX = 32, 12
CODES_HIST = 2 * (RED_CTX + DEC_CTX)


def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    new = ("fac_vc_stream_set_timbre", "fac_vc_pool_set_timbre", "fac_vc_pool_open_mode")
    assert set(new) <= set(_declared("facodec_b200.h"))
    assert "fac_debug_vc_plan" in _declared("facodec_b200_debug.h")
    assert set(new) | {"fac_debug_vc_plan"} <= set(_lib.EXPORTED)


# ---------------------------------------------------------------------------------------------------------------------
# host: the step plan
# ---------------------------------------------------------------------------------------------------------------------
def plan_restated(N, Zf, Yf, F, finish, stale):
    """The 16 integers of fac_debug_vc_plan, restated."""
    f0 = lambda v: max(v, 0)
    N1 = N + F
    Zf1 = N1 if finish else max(N1 - RED_CTX, Zf)
    Yf1 = N1 if finish else max(Zf1 - DEC_CTX, Yf)
    zh0, zh1 = f0(Yf - DEC_CTX), f0(Yf1 - DEC_CTX)
    stale = int(bool(stale) and Zf > zh0)
    hc0 = f0(zh0 - RED_CTX) if stale else f0(Zf - RED_CTX)
    z0 = zh0 if stale else Zf
    return [F, N1 - hc0, N - hc0, Zf1 - zh0, z0 - zh0, z0 - hc0, Zf1 - z0, Yf1 - Yf, Yf - zh0, zh1 - zh0, Zf1 - zh1, stale,
            N1, Zf1, Yf1, CODES_HIST]


def plan_engine(N, Zf, Yf, F, finish, stale):
    from facodec_b200 import _lib
    out = np.zeros(16, dtype=np.int64)
    assert _lib.load().fac_debug_vc_plan(N, Zf, Yf, F, int(finish), int(stale), out.ctypes.data_as(ctypes.c_void_p)) == 16
    return [int(v) for v in out]


@pytest.mark.parametrize("seed", range(4))
def test_stale_plan_matches_restatement(seed, built_lib):
    rng = random.Random(300 + seed)
    for _ in range(2000):
        N = rng.choice([0, 1, 5, 31, 32, 33, 44, 45, 56, 57, 88, 89]) if rng.random() < 0.3 else rng.randint(0, 5000)
        Zf = rng.randint(0, N)
        Yf = rng.randint(0, Zf)
        finish = rng.random() < 0.2
        F = 0 if finish else rng.choice([1, 7, 20, 37, rng.randint(1, 300)])
        stale = rng.random() < 0.5
        assert plan_engine(N, Zf, Yf, F, finish, stale) == plan_restated(N, Zf, Yf, F, finish, stale), (N, Zf, Yf, F, finish, stale)
    from facodec_b200 import _lib
    out = np.zeros(16, dtype=np.int64)
    for bad in ((10, 0, 0, 0, 0, 0), (10, 0, 0, 5, 1, 0), (10, 0, 0, -1, 0, 0)):
        assert _lib.load().fac_debug_vc_plan(*bad, out.ctypes.data_as(ctypes.c_void_p)) == -1


@pytest.mark.parametrize("seed", range(4))
def test_codes_history_bound_on_random_walks(seed, built_lib):
    """Streams stepped by random chunks with random switches: every step reads at most CODES_HIST frames of code history,
    and after every step the history a switch would need, [max(0, Yf - 12 - 32), N), fits in it.  The z window reads only
    rows the stream keeps, and a stale step re-reads the whole z window from codes."""
    rng = random.Random(400 + seed)
    for _ in range(30):
        N = Zf = Yf = 0
        kept_z = (0, 0)                                      # z rows [lo, hi) the stream holds
        for _ in range(rng.randint(1, 200)):
            finish = rng.random() < 0.02
            F = 0 if finish else rng.choice([1, 1, 7, 20, 37, rng.randint(1, 120)])
            stale = rng.random() < 0.3
            p = plan_engine(N, Zf, Yf, F, finish, stale)
            Fp, Tw, hist, Tz, zhist, zoff, znew, k, yoff, zkeep_at, zkeep, st, N1, Zf1, Yf1, cap = p
            assert cap == CODES_HIST and 0 <= hist <= cap and Tw == hist + F
            assert 0 <= zhist <= 2 * DEC_CTX and (zhist == 0 or kept_z == (Zf - zhist, Zf))
            if st:
                assert zhist == 0 and znew == Tz and zoff + znew <= Tw
            assert N1 - max(Yf1 - DEC_CTX - RED_CTX, 0) <= cap
            assert 0 <= zkeep <= 2 * DEC_CTX
            kept_z = (Zf1 - zkeep, Zf1)
            N, Zf, Yf = N1, Zf1, Yf1
            if finish:
                assert N == Zf == Yf
                break


def pool_plan(counters, lengths, kind):
    from facodec_b200 import _lib
    n = len(lengths)
    c = np.ascontiguousarray(np.array(counters, dtype=np.int64).reshape(-1))
    ln = np.array(lengths, dtype=np.int32)
    group, batch = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    nb = _lib.load().fac_debug_pool_plan(kind, n, P(c), P(ln), P(group), P(batch))
    assert nb >= 0
    return list(group), list(batch), nb


@pytest.mark.parametrize("seed", range(4))
def test_vc_pool_plan_with_switches(seed, built_lib):
    """Switched sessions group among themselves; unswitched ones group exactly as a pool without switches does."""
    from test_stream_pool import plan_restated as grouping, vc_counters
    rng = random.Random(500 + seed)
    n = rng.choice([9, 50, 80])
    base = [vc_counters(rng.choice([0, 1, 20, 40, 44, 60]) if rng.random() < 0.3 else rng.randint(70, 900)) for _ in range(n)]
    stale = [int(rng.random() < 0.25) for _ in range(n)]
    lengths = [rng.choice([20] * 5 + [1, 7, 13, 50]) for _ in range(n)]
    keys = [tuple(plan_restated(*c, F, False, s)[:12]) for c, F, s in zip(base, lengths, stale)]
    got = pool_plan([list(c) + [s] for c, s in zip(base, stale)], lengths, 3)
    assert got == grouping(keys)
    group = got[0]
    plain = pool_plan([list(c) + [0] for c in base], lengths, 3)
    assert plain == pool_plan(base, lengths, 1)
    for i in range(n):
        for j in range(n):
            ei, ej = keys[i][11], keys[j][11]                     # effective staleness (a non-empty z history)
            if ei != ej:
                assert group[i] != group[j]
            elif not ei and plain[0][i] == plain[0][j]:
                assert group[i] == group[j]


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _codes(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 1024, (B, 1, T), generator=g).cuda(), torch.randint(0, 1024, (B, 2, T), generator=g).cuda()


def _timbres(B, n, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, 1024, generator=g).cuda() for _ in range(n)]


def _splice(offline, pieces):
    """pieces: (timbre index, output frames) in emission order -> the spliced waveform [B,1,300 sum]."""
    out, f = [], 0
    for t, k in pieces:
        out.append(offline[t][:, :, 300 * f:300 * (f + k)])
        f += k
    return torch.cat(out, dim=2)


def _switch_rule(T):
    """Before a call at (N, Zf, Yf): the timbre index to switch to (a list: several switches in a row), or None.  Switches:
    before the first call; with Yf = 0 and Zf > 0; on the first call after the look-ahead fills; twice in a row in mid
    utterance, ending on the original voice; to the voice already active; and before finish."""
    fired = set()

    def rule(N, Zf, Yf, last):
        for name, cond, to in (("start", N == 0, [1]), ("zf", Zf > 0 and Yf == 0, [2]), ("filled", Yf > 0, [1]),
                               ("mid", N >= T // 2, [2, 0]), ("same", N >= 3 * T // 4, [0]), ("finish", last, [1])):
            if cond and name not in fired:
                fired.add(name)
                return to
        return None
    return rule


def _run_stream(m, cp, cc, timbres, sizes, mode=dict(use_p_code=False, n_c=1), switches=True):
    """A VoiceConversionStream over the codes in chunks of `sizes` with the switches of _switch_rule -> (output, pieces)."""
    import facodec_b200 as fb
    from test_gpu_stream import chunks_of
    T = cp.shape[2]
    rule = _switch_rule(T)
    cur, outs, pieces = 0, [], []
    N = 0
    with fb.VoiceConversionStream(m, cp.shape[0], timbres[0], **mode) as vs:
        for p, n in chunks_of(T, sizes):
            Zf = max(N - RED_CTX, 0)
            to = rule(N, Zf, max(Zf - DEC_CTX, 0), False) if switches else None
            for t in to or []:
                vs.set_timbre(timbres[t])
                cur = t
            y = vs.convert([cp[:, :, p:p + n], cc[:, :, p:p + n]])
            outs.append(y)
            pieces.append((cur, y.shape[2] // 300))
            N += n
        to = rule(N, 0, 0, True) if switches else None
        for t in to or []:
            vs.set_timbre(timbres[t])
            cur = t
        y = vs.finish()
        outs.append(y)
        pieces.append((cur, y.shape[2] // 300))
    return torch.cat(outs, dim=2), pieces


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 7, 20, 37])
def test_stream_switch_is_a_splice_of_offline_conversions(size, built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    T = 1700 + 13 * size                                     # 21-27 s of codes
    cp, cc = _codes(1, T, 600 + size)
    timbres = _timbres(1, 3, 700 + size)
    y, pieces = _run_stream(m, cp, cc, timbres, [size])
    assert len({t for t, k in pieces if k}) == 3             # every voice reached the output
    offline = [fb.VoiceConverter(m).convert([cp, cc], tv, use_p_code=False, n_c=1) for tv in timbres]
    assert torch.equal(y, _splice(offline, pieces))
    assert not torch.equal(y, offline[0])


@pytest.mark.gpu
def test_stream_switch_batch_rows_together(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    cp, cc = _codes(3, 1800, 801)
    timbres = _timbres(3, 3, 802)
    for mode in (dict(use_p_code=False, n_c=1), dict(use_p_code=True, n_c=2)):
        y, pieces = _run_stream(m, cp, cc, timbres, [20, 7, 37], mode=mode)
        offline = [fb.VoiceConverter(m).convert([cp, cc], tv, **mode) for tv in timbres]
        assert torch.equal(y, _splice(offline, pieces))


MODES = [(0, 1), (1, 1), (0, 2), (1, 2)]


def _lockstep(pool, sessions, cps, ccs, sizes, on_step=None):
    """Feeds every session the same chunking in lockstep, then finishes them -> ({session: output}, launch counts)."""
    from test_gpu_stream import chunks_of
    outs, counts = {s: [] for s in sessions}, []
    e = pool.engine
    for k, (p, n) in enumerate(chunks_of(cps[0].shape[2], sizes)):
        if on_step:
            on_step(k)
        got = pool.convert({s: [cps[i][:, :, p:p + n], ccs[i][:, :, p:p + n]] for i, s in enumerate(sessions)})
        counts.append(e.L.fac_last_launch_count(e.handle))
        for s in sessions:
            outs[s].append(got[s])
    for s, y in pool.finish(sessions).items():
        outs[s].append(y)
    return {s: torch.cat(v, dim=2) for s, v in outs.items()}, counts


@pytest.mark.gpu
def test_mixed_modes_share_one_launch_sequence(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    T = 400
    codes = [_codes(1, T, 900 + i) for i in range(8)]
    cps, ccs = [c[0] for c in codes], [c[1] for c in codes]
    tvs = _timbres(1, 8, 901)
    sizes = [20, 7, 37, 1, 20]
    with fb.VoiceConversionPool(m, capacity=8, use_p_code=False, use_c_code=True, n_c=1) as pool:
        sess = [pool.open(tvs[i], use_p_code=bool(MODES[i % 4][0]), n_c=MODES[i % 4][1]) for i in range(8)]
        mixed, n_mixed = _lockstep(pool, sess, cps, ccs, sizes)
    with fb.VoiceConversionPool(m, capacity=8, use_p_code=False, use_c_code=True, n_c=1) as pool:
        sess_u = [pool.open(tvs[i]) for i in range(8)]
        _, n_uniform = _lockstep(pool, sess_u, cps, ccs, sizes)
    assert n_mixed == n_uniform                       # one shared sequence per step, not one per mode
    for i in range(8):
        use_p, n_c = MODES[i % 4]
        with fb.VoiceConversionStream(m, 1, tvs[i], use_p_code=bool(use_p), n_c=n_c) as vs:
            from test_gpu_stream import chunks_of
            ref = [vs.convert([cps[i][:, :, p:p + n], ccs[i][:, :, p:p + n]]) for p, n in chunks_of(T, sizes)]
            ref.append(vs.finish())
        assert torch.equal(mixed[sess[i]], torch.cat(ref, dim=2)), i
        off = fb.VoiceConverter(m).convert([cps[i], ccs[i]], tvs[i], use_p_code=bool(use_p), n_c=n_c)
        assert torch.equal(mixed[sess[i]], off), i
    # use_c_code = False (no content embedding) in the same batch
    with fb.VoiceConversionPool(m, capacity=2, n_c=1) as pool:
        a, b = pool.open(tvs[0]), pool.open(tvs[1], use_p_code=True, use_c_code=False, n_c=2)
        got, _ = _lockstep(pool, [a, b], cps[:2], ccs[:2], [20])
    assert torch.equal(got[b], fb.VoiceConverter(m).convert([cps[1], ccs[1]], tvs[1], use_p_code=True, use_c_code=False, n_c=2))
    assert torch.equal(got[a], fb.VoiceConverter(m).convert([cps[0], ccs[0]], tvs[0], use_p_code=False, n_c=1))


@pytest.mark.gpu
def test_switch_in_a_pool(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    T = 600
    codes = [_codes(1, T, 1000 + i) for i in range(4)]
    cps, ccs = [c[0] for c in codes], [c[1] for c in codes]
    tvs = _timbres(1, 4, 1001)
    new = _timbres(1, 1, 1002)[0]
    with fb.VoiceConversionPool(m, capacity=4, n_c=1) as pool:
        sess = [pool.open(tvs[i], n_c=1 + i % 2) for i in range(4)]
        plain, _ = _lockstep(pool, sess, cps, ccs, [20])
    with fb.VoiceConversionPool(m, capacity=4, n_c=1) as pool:
        sess = [pool.open(tvs[i], n_c=1 + i % 2) for i in range(4)]
        got, _ = _lockstep(pool, sess, cps, ccs, [20], on_step=lambda k: pool.set_timbre(sess[1], new) if k == 12 else None)
    for i in (0, 2, 3):
        assert torch.equal(got[sess[i]], plain[sess[i]]), i
    # session 1 switched before its 13th chunk of 20 frames: N = 240, Yf = 240 - 44
    off = [fb.VoiceConverter(m).convert([cps[1], ccs[1]], tv, use_p_code=False, n_c=2) for tv in (tvs[1], new)]
    Yf = 240 - RED_CTX - DEC_CTX
    assert torch.equal(got[sess[1]], torch.cat([off[0][:, :, :300 * Yf], off[1][:, :, 300 * Yf:]], dim=2))
    assert not torch.equal(got[sess[1]], plain[sess[1]])


@pytest.mark.gpu
def test_switch_at_48k(built_lib):
    import facodec_b200 as fb
    from test_gpu_parity import redec_model_for
    from test_gpu_stream import chunks_of
    m = redec_model_for(0)
    T = 500
    (cp, cc), (cp2, cc2) = _codes(1, T, 1100), _codes(1, T, 1101)
    tv, new, tv2 = _timbres(1, 3, 1102)
    outs = {0: [], 1: []}
    with fb.VoiceConversionPool(m, capacity=2, n_c=1) as pool:
        a, b = pool.open(tv, sample_rate=48000), pool.open(tv2)
        for k, (p, n) in enumerate(chunks_of(T, [20, 7])):
            if k == 9:
                pool.set_timbre(a, new)
            got = pool.convert({a: [cp[:, :, p:p + n], cc[:, :, p:p + n]], b: [cp2[:, :, p:p + n], cc2[:, :, p:p + n]]})
            outs[0].append(got[a].view(-1)); outs[1].append(got[b].view(-1))
        fin = pool.finish([a, b])
        outs[0].append(fin[a].view(-1)); outs[1].append(fin[b].view(-1))
    N = sum(n for _, n in chunks_of(T, [20, 7])[:9])
    Yf = N - RED_CTX - DEC_CTX
    off = [fb.VoiceConverter(m).convert([cp, cc], t, use_p_code=False, n_c=1) for t in (tv, new)]
    splice = torch.cat([off[0][:, :, :300 * Yf], off[1][:, :, 300 * Yf:]], dim=2)
    assert torch.equal(torch.cat(outs[0]), fb.resample(splice, 24000, 48000).view(-1))
    assert torch.equal(torch.cat(outs[1]), fb.VoiceConverter(m).convert([cp2, cc2], tv2, use_p_code=False, n_c=1).view(-1))


@pytest.mark.gpu
def test_rejected_calls_change_nothing(built_lib):
    import facodec_b200 as fb
    from facodec_b200.modules import _ptr, _stream
    from test_gpu_parity import redec_model_for
    m = redec_model_for(0)
    T = 200
    codes = [_codes(1, T, 1200 + i) for i in range(3)]
    tvs = _timbres(1, 3, 1201)
    part = lambda i, lo, hi: [codes[i][0][:, :, lo:hi], codes[i][1][:, :, lo:hi]]
    e = fb.VoiceConverter(m).engine
    with fb.VoiceConversionPool(m, capacity=4, n_c=1) as pool:
        s = [pool.open(tvs[i]) for i in range(3)]
        ys = {x: [] for x in s}
        for x, y in pool.convert({s[i]: part(i, 0, 100) for i in range(3)}).items():
            ys[x].append(y)
        closed = pool.open(tvs[0])
        pool.close(closed)
        with pytest.raises(ValueError):
            pool.set_timbre(s[0], torch.randn(1, 512, device="cuda"))         # wrong shape
        with pytest.raises(ValueError):
            pool.set_timbre(s[0], torch.randn(2, 1024, device="cuda"))
        with pytest.raises(fb.FacError):
            pool.set_timbre(s[1], torch.randn(1, 1024))                        # another device
        with pytest.raises(fb.FacError):
            pool.set_timbre(closed, tvs[1])                                    # closed
        with pytest.raises(ValueError):
            pool.open(tvs[1], n_c=3)
        assert e.L.fac_vc_pool_open_mode(e.handle, pool.pid, _ptr(tvs[1]), 0, 1, 3, _stream(tvs[1].device)) == -1
        assert e.L.fac_vc_pool_set_timbre(e.handle, pool.pid, s[0], None, _stream(tvs[1].device)) == -1
        assert e.L.fac_vc_pool_set_timbre(e.handle, pool.pid, closed, _ptr(tvs[1]), _stream(tvs[1].device)) == -1
        for x, y in pool.convert({s[i]: part(i, 100, T) for i in range(3)}).items():
            ys[x].append(y)
        for x, y in pool.finish([s[2]]).items():
            ys[x].append(y)
        with pytest.raises(fb.FacError):
            pool.set_timbre(s[2], tvs[0])                                      # finished
        assert e.L.fac_vc_pool_set_timbre(e.handle, pool.pid, s[2], _ptr(tvs[0]), _stream(tvs[0].device)) == -2
        for x, y in pool.finish(s[:2]).items():
            ys[x].append(y)
    for i in range(3):
        off = fb.VoiceConverter(m).convert([codes[i][0], codes[i][1]], tvs[i], use_p_code=False, n_c=1)
        assert torch.equal(torch.cat(ys[s[i]], dim=2), off), i

    cp, cc = codes[0]
    with fb.VoiceConversionStream(m, 1, tvs[0], use_p_code=False, n_c=1) as vs:
        y = [vs.convert([cp[:, :, :120], cc[:, :, :120]])]
        with pytest.raises(ValueError):
            vs.set_timbre(torch.randn(1, 100, device="cuda"))
        with pytest.raises(fb.FacError):
            vs.set_timbre(torch.randn(1, 1024))
        assert e.L.fac_vc_stream_set_timbre(e.handle, vs.sid, None, _stream(cp.device)) == -1
        y.append(vs.convert([cp[:, :, 120:], cc[:, :, 120:]]))
        y.append(vs.finish())
        with pytest.raises(fb.FacError):
            vs.set_timbre(tvs[1])                                              # finished
        sid = vs.sid
    with pytest.raises(fb.FacError):
        vs.set_timbre(tvs[1])                                                  # closed
    assert e.L.fac_vc_stream_set_timbre(e.handle, sid, _ptr(tvs[1]), _stream(cp.device)) == -1
    assert torch.equal(torch.cat(y, dim=2), fb.VoiceConverter(m).convert([cp, cc], tvs[0], use_p_code=False, n_c=1))
