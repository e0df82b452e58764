"""Moving live pool sessions between pools, handles and devices (fac_*_pool_export_size / _export / _import;
SessionState, <Pool>.export / import_session).

Every GPU comparison is torch.equal against a twin session that never moved and is fed the same chunks: after an import
the session continues bit for bit, in the same pool, another pool, another engine built from the same state dicts, through
to_bytes / from_bytes, or on cuda:1.  The source session keeps running unchanged (export is read-only), two imports of one
state both continue (a fork), an imported session shares batches with native ones at the launch counts of a pool where
nothing moved, and every rejected import changes neither pool.  On the host: the header layout and its checks."""
import ctypes
import struct

import numpy as np
import pytest
import torch

MAGIC, VERSION = 0x54534346, 1
HEADER = struct.Struct("<4IQ12q12q6qQQ")          # magic, version, kind, header_bytes, fingerprint, options, counters,
                                                  # region_bytes, payload_bytes, checksum
NEW = [f"fac_{k}_pool_{op}" for k in ("codes", "vc", "dec", "rs") for op in ("export_size", "export", "import")]


def test_new_entry_points_registered():
    from facodec_b200 import _lib
    from test_host import _declared
    assert set(NEW) <= set(_declared("facodec_b200.h"))
    assert "fac_debug_state_header" in _declared("facodec_b200_debug.h")
    assert set(NEW) | {"fac_debug_state_header"} <= set(_lib.EXPORTED)


# ---------------------------------------------------------------------------------------------------------------------
# host: the header
# ---------------------------------------------------------------------------------------------------------------------
def fnv1a(b):
    h = 14695981039346656037
    for x in b:
        h = ((h ^ x) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def make_header(kind=1, fp=0x1234, options=(2, 1, 1, 1, 0, 1, 1, 0, 0, 1, 1), counters=(2, 2, 6000, 19, 6000, 2),
                regions=(24000, 8192, 4096, 16384, 6080), version=VERSION, magic=MAGIC, size=None, payload=None):
    opts = list(options) + [0] * (12 - len(options))
    ctr = list(counters) + [0] * (12 - len(counters))
    reg = list(regions) + [0] * (6 - len(regions))
    body = HEADER.pack(magic, version, kind, HEADER.size if size is None else size, fp, *opts, *ctr, *reg,
                       sum(regions) if payload is None else payload, 0)
    return body[:-8] + struct.pack("<Q", fnv1a(body[:-8]))


def check_header(hdr, kind=1, fp=0x1234, options=(2, 1, 1, 1, 0, 1, 1, 0, 0, 1, 1), payload_bytes=None):
    from facodec_b200 import _lib
    L = _lib.load()
    opts = np.zeros(12, dtype=np.int64)
    opts[:len(options)] = options
    out = np.zeros(12, dtype=np.int64)
    if payload_bytes is None:
        payload_bytes = HEADER.unpack(hdr[:HEADER.size])[-2] if len(hdr) >= HEADER.size else 0
    buf = ctypes.create_string_buffer(hdr, len(hdr))
    L.fac_debug_state_header.restype = ctypes.c_int
    rc = L.fac_debug_state_header(buf, ctypes.c_size_t(len(hdr)), kind, ctypes.c_uint64(fp),
                                  opts.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(payload_bytes),
                                  out.ctypes.data_as(ctypes.c_void_p))
    return rc, [int(v) for v in out]


def test_header_layout_and_checks(built_lib):
    assert HEADER.size == 280
    hdr = make_header()
    rc, counters = check_header(hdr)
    assert rc == 0 and counters[:6] == [2, 2, 6000, 19, 6000, 2]
    assert check_header(hdr[:-1])[0] == -1                                  # truncated
    assert check_header(hdr + b"\0")[0] == -1                               # longer than the struct
    for byte in (0, 9, 40, 200, 270):                                       # any flipped bit breaks the checksum
        bad = bytearray(hdr)
        bad[byte] ^= 0x10
        assert check_header(bytes(bad))[0] == -1, byte
    assert check_header(make_header(magic=0x12345678))[0] == -1
    assert check_header(make_header(size=272))[0] == -1
    assert check_header(make_header(version=2))[0] == -2                    # another format version
    assert check_header(hdr, kind=3)[0] == -1                               # another pool kind
    assert check_header(hdr, fp=0x1235)[0] == -2                            # other weights
    assert check_header(hdr, options=(2, 1, 1, 1, 1, 1, 1, 0, 0, 1, 1))[0] == -2
    assert check_header(hdr, payload_bytes=sum((24000, 8192, 4096, 16384, 6080)) - 4)[0] == -1
    assert check_header(make_header(payload=100))[0] == -1                  # regions disagree with payload_bytes
    assert check_header(make_header(regions=(24000, 8192, 4096, 16384, 6082)))[0] == -1   # not whole words
    assert check_header(make_header(regions=(24000, -4, 4096, 16384, 6080)))[0] == -1


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _eq(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_eq(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_eq(x, y) for x, y in zip(a, b))
    return torch.equal(a, b)


def _codec(seed=0, fresh=False):
    import facodec_b200 as fb
    from facodec_b200 import synth
    if not fresh:
        from test_gpu_parity import model_for
        return model_for(seed)
    m = fb.build_model()
    sds = synth.synth_state_dicts(seed)
    for k in ("encoder", "quantizer", "decoder"):
        m[k].load_state_dict(sds[k])
        m[k].eval()
    return m


def _redec(seed=0, fresh=False):
    import facodec_b200 as fb
    from facodec_b200 import synth
    if not fresh:
        from test_gpu_parity import redec_model_for
        return redec_model_for(seed)
    m = fb.build_model(stage="redecoder")
    sds = synth.synth_redecoder_state_dicts(seed)
    for k in ("encoder", "decoder"):
        m[k].load_state_dict(sds[k])
        m[k].eval()
    return m


def _wave(T, seed, device="cuda:0"):
    from facodec_b200 import synth
    return synth.synth_waves(1, T, seed=seed).to(device)


def _feeds(total, sizes, cut):
    from test_gpu_stream import chunks_of
    return [cut(p, n) for p, n in chunks_of(total, sizes)]


class Kind:
    """How to open, feed and finish sessions of one pool kind."""

    def __init__(self, open_fn, step, finish, feeds):
        self.open, self.step, self.finish, self.feeds = open_fn, step, finish, feeds


def _codes_kind(sizes=(3000, 300, 900, 6000), T=300 * 160, seed=1, sample_rate=24000):
    x = _wave(T, seed)
    return Kind(lambda p: p.open(sample_rate=sample_rate), lambda p, f: p.encode_codes(f), lambda p, s: p.finish_codes(s),
                lambda dev="cuda:0": _feeds(T, list(sizes), lambda q, n: x[:, :, q:q + n].to(dev)))


def _vc_kind(timbre, sizes=(20, 7, 37, 1, 20), T=400, seed=5, mode=None, sample_rate=24000):
    g = torch.Generator().manual_seed(seed)
    cp, cc = torch.randint(0, 1024, (1, 1, T), generator=g), torch.randint(0, 1024, (1, 2, T), generator=g)
    return Kind(lambda p: p.open(timbre.to(p.device), sample_rate=sample_rate, **(mode or {})), lambda p, f: p.convert(f),
                lambda p, s: p.finish(s),
                lambda dev="cuda:0": _feeds(T, list(sizes), lambda q, n: [cp[:, :, q:q + n].to(dev), cc[:, :, q:q + n].to(dev)]))


def _dec_kind(timbre, sizes=(10, 3, 7, 25), T=160, seed=6, sample_rate=24000):
    g = torch.Generator().manual_seed(seed)
    codes = [torch.randint(0, 1024, (1, r, T), generator=g) for r in (1, 2, 3)]
    return Kind(lambda p: p.open(timbre.to(p.device), sample_rate=sample_rate), lambda p, f: p.decode_codes(f),
                lambda p, s: p.finish(s),
                lambda dev="cuda:0": _feeds(T, list(sizes), lambda q, n: [c[:, :, q:q + n].to(dev) for c in codes]))


def _rs_kind(orig=48000, new=24000, sizes=(1000, 7, 480, 3333), T=30000, seed=7):
    x = _wave(T, seed)
    return Kind(lambda p: p.open(orig, new), lambda p, f: p.push(f), lambda p, s: p.finish(s),
                lambda dev="cuda:0": _feeds(T, list(sizes), lambda q, n: x[0, 0, q:q + n].to(dev)))


def _to_dev(out, dev):
    if isinstance(out, dict):
        return {k: _to_dev(v, dev) for k, v in out.items()}
    if isinstance(out, (list, tuple)):
        return type(out)(_to_dev(v, dev) for v in out)
    return out.to(dev)


def move_and_compare(kind, src, dst, export_at, via=lambda st: st, before_export=None, extra=None):
    """Opens session a and its twin t in src and feeds both; before feed `export_at` (== len(feeds): before finish) it
    exports a, passes the state through `via` and imports it into dst as b.  From then on a, t and b take the same feeds and
    every output of a and b equals t's.  before_export(pool, a, t) runs on the source pair first (e.g. a switch);
    extra(pool, session) -> output is compared after every step once b exists (e.g. the timbre so far)."""
    a, t = kind.open(src), kind.open(src)
    feeds = kind.feeds()
    dev = dst.device
    b = None
    for k in range(len(feeds) + 1):
        if k == export_at:
            if before_export:
                before_export(src, a, t)
            b = dst.import_session(via(src.export([a])[a]))
        if k == len(feeds):
            break
        out = kind.step(src, {a: feeds[k], t: feeds[k]})
        assert _eq(out[a], out[t]), ("source after export", k)
        if b is not None:
            got = kind.step(dst, {b: feeds[k].to(dev) if torch.is_tensor(feeds[k]) else [f.to(dev) for f in feeds[k]]})
            assert _eq(_to_dev(got[b], "cpu"), _to_dev(out[t], "cpu")), ("imported", k)
            if extra:
                assert _eq(_to_dev(extra(dst, b), "cpu"), _to_dev(extra(src, t), "cpu")), ("extra", k)
    fin = kind.finish(src, [a, t])
    assert _eq(fin[a], fin[t])
    got = kind.finish(dst, [b])
    assert _eq(_to_dev(got[b], "cpu"), _to_dev(fin[t], "cpu"))
    for p, s in ((src, a), (src, t), (dst, b)):
        p.close(s)


def _codes_timbre(p, s):
    return p.timbre([s])[s]


def _targets(make_pool, other_model, make_other_engine_pool):
    """Import targets by name: src -> (target pool, what the state passes through).  The second engine is built once."""
    import facodec_b200 as fb
    built = []
    other = lambda: built[0] if built else built.append(other_model()) or built[0]
    return {
        "same": lambda src: (src, lambda st: st),
        "other_pool": lambda src: (make_pool(3), lambda st: st),
        "other_engine": lambda src: (make_other_engine_pool(other()), lambda st: st),
        "bytes": lambda src: (src, lambda st: fb.SessionState.from_bytes(st.to_bytes())),
    }


TARGETS = ["same", "other_pool", "other_engine", "bytes"]


@pytest.mark.gpu
@pytest.mark.parametrize("target", TARGETS)
def test_codes_pool_moves(target, built_lib):
    import facodec_b200 as fb
    m = _codec()
    src = fb.CodecStreamPool(m, capacity=8, n_c=2)
    tgt = _targets(lambda cap: fb.CodecStreamPool(m, capacity=cap, n_c=2),
                   lambda: _codec(fresh=True), lambda om: fb.CodecStreamPool(om, capacity=4, n_c=2))[target]
    kind = _codes_kind()
    n = len(kind.feeds())
    for at in (0, 1, 2, 8, n):               # before any chunk, after the first, in the first 20 frames, steady, before finish
        dst, via = tgt(src)
        move_and_compare(kind, src, dst, at, via, extra=_codes_timbre if at in (2, 8) else None)


@pytest.mark.gpu
@pytest.mark.parametrize("target", TARGETS)
def test_vc_pool_moves(target, built_lib):
    import facodec_b200 as fb
    m = _redec()
    g = torch.Generator().manual_seed(20)
    tv, tv2 = torch.randn(1, 1024, generator=g).cuda(), torch.randn(1, 1024, generator=g).cuda()
    src = fb.VoiceConversionPool(m, capacity=8, n_c=1)
    tgt = _targets(lambda cap: fb.VoiceConversionPool(m, capacity=cap, n_c=1),
                   lambda: _redec(fresh=True), lambda om: fb.VoiceConversionPool(om, capacity=4, n_c=1))[target]
    for at in (0, 1, 2, 8):                   # 20 + 7 frames: the 44-frame look-ahead is not full yet at 2
        dst, via = tgt(src)
        move_and_compare(_vc_kind(tv), src, dst, at, via)
    switch = lambda p, a, t: (p.set_timbre(a, tv2), p.set_timbre(t, tv2))
    for at in (0, 3, 9):                      # exported stale, right after the switch
        dst, via = tgt(src)
        move_and_compare(_vc_kind(tv), src, dst, at, via, before_export=switch)
    dst, via = tgt(src)                       # a non-default mode
    move_and_compare(_vc_kind(tv, mode=dict(use_p_code=True, n_c=2)), src, dst, 4, via)


@pytest.mark.gpu
@pytest.mark.parametrize("target", TARGETS)
def test_dec_pool_moves(target, built_lib):
    import facodec_b200 as fb
    m = _codec()
    g = torch.Generator().manual_seed(21)
    tv, tv2 = torch.randn(1, 1024, generator=g).cuda(), torch.randn(1, 1024, generator=g).cuda()
    src = fb.CodecDecodePool(m, capacity=8)
    tgt = _targets(lambda cap: fb.CodecDecodePool(m, capacity=cap),
                   lambda: _codec(fresh=True), lambda om: fb.CodecDecodePool(om, capacity=4))[target]
    for at in (0, 1, 2, 9):                   # 10 + 3 frames: within the first 20 at 2
        dst, via = tgt(src)
        move_and_compare(_dec_kind(tv), src, dst, at, via)
    dst, via = tgt(src)                       # gamma | beta of a set_timbre travel with the state
    move_and_compare(_dec_kind(tv), src, dst, 5, via, before_export=lambda p, a, t: (p.set_timbre(a, tv2), p.set_timbre(t, tv2)))


@pytest.mark.gpu
@pytest.mark.parametrize("target", ["same", "other_pool", "bytes"])
def test_resample_pool_moves(target, built_lib):
    import facodec_b200 as fb
    src = fb.ResamplePool(capacity=4)
    tgt = {"same": (src, lambda st: st), "other_pool": (fb.ResamplePool(capacity=2, device="cuda:0"), lambda st: st),
           "bytes": (src, lambda st: fb.SessionState.from_bytes(st.to_bytes()))}[target]
    for orig, new in ((48000, 24000), (24000, 16000), (24000, 24000)):
        for at in (0, 1, 3):
            move_and_compare(_rs_kind(orig, new), src, tgt[0], at, tgt[1])


@pytest.mark.gpu
def test_codes_pool_move_after_60_s(built_lib):
    """A large mel history: 60 s in 1 s chunks, exported at 60 s (~1.9 MB payload), imported into another engine."""
    import facodec_b200 as fb
    m = _codec()
    T = 24000 * 64
    kind = _codes_kind(sizes=(24000,), T=T, seed=3)
    src = fb.CodecStreamPool(m, capacity=4, n_c=2)
    dst = fb.CodecStreamPool(_codec(fresh=True), capacity=2, n_c=2)
    move_and_compare(kind, src, dst, 60, lambda st: fb.SessionState.from_bytes(st.cpu().to_bytes()), extra=_codes_timbre)


@pytest.mark.gpu
def test_vc_and_dec_moves_after_60_s(built_lib):
    import facodec_b200 as fb
    g = torch.Generator().manual_seed(22)
    tv = torch.randn(1, 1024, generator=g).cuda()
    src = fb.VoiceConversionPool(_redec(), capacity=4, n_c=1)
    move_and_compare(_vc_kind(tv, sizes=(80,), T=80 * 64), src, src, 60, lambda st: st)
    src = fb.CodecDecodePool(_codec(), capacity=4)
    move_and_compare(_dec_kind(tv, sizes=(80,), T=80 * 64), src, src, 60, lambda st: st)


@pytest.mark.gpu
def test_export_is_read_only_and_forks(built_lib):
    """Two imports of one state both continue bit for bit, next to the source session that keeps running."""
    import facodec_b200 as fb
    m = _codec()
    kind = _codes_kind()
    feeds = kind.feeds()
    with fb.CodecStreamPool(m, capacity=8, n_c=2) as pool:
        a, t = pool.open(), pool.open()
        for f in feeds[:4]:
            pool.encode_codes({a: f, t: f})
        st = pool.export([a])[a]
        b, c = pool.import_session(st), pool.import_session(st)
        for f in feeds[4:]:
            out = pool.encode_codes({a: f, t: f, b: f, c: f})
            assert _eq(out[a], out[t]) and _eq(out[b], out[t]) and _eq(out[c], out[t])
        fin = pool.finish_codes([a, t, b, c])
        assert _eq(fin[a], fin[t]) and _eq(fin[b], fin[t]) and _eq(fin[c], fin[t])


def _launches(pool):
    e = pool.engine
    return e.L.fac_last_launch_count(e.handle)


@pytest.mark.gpu
def test_imported_session_shares_batches(built_lib):
    """Pool dst holds 3 native sessions; a 4th with the same progress moves in from src.  Every step of dst then runs the
    launches, and gives the outputs, of a pool where the same 4 sessions never moved."""
    import facodec_b200 as fb
    m = _codec()
    xs = [_wave(300 * 120, 40 + i) for i in range(4)]
    sizes = [3000, 900, 6000, 900, 6000, 6000, 6000, 3000, 4200]
    from test_gpu_stream import chunks_of
    steps = chunks_of(300 * 120, sizes)
    ref, ref_n = [], []
    with fb.CodecStreamPool(m, capacity=4, n_c=2) as pool:
        s = [pool.open() for _ in range(4)]
        for p, n in steps:
            ref.append(pool.encode_codes({s[i]: xs[i][:, :, p:p + n] for i in range(4)}))
            ref_n.append(_launches(pool))
        ref_fin = pool.finish_codes(s)
        ref = [{i: r[s[i]] for i in range(4)} for r in ref]
        ref_fin = {i: ref_fin[s[i]] for i in range(4)}
    with fb.CodecStreamPool(m, capacity=4, n_c=2) as src, fb.CodecStreamPool(m, capacity=5, n_c=2) as dst:
        d = [dst.open() for _ in range(3)]
        a = src.open()
        for k, (p, n) in enumerate(steps):
            if k == 3:
                old = a
                a = dst.import_session(src.export([old])[old])
                src.close(old)
                d.append(a)
            if k < 3:
                out3 = dst.encode_codes({d[i]: xs[i][:, :, p:p + n] for i in range(3)})
                out1 = src.encode_codes({a: xs[3][:, :, p:p + n]})
                out = {**{i: out3[d[i]] for i in range(3)}, 3: out1[a]}
            else:
                got = dst.encode_codes({d[i]: xs[i][:, :, p:p + n] for i in range(4)})
                assert _launches(dst) == ref_n[k], k
                out = {i: got[d[i]] for i in range(4)}
            assert _eq(out, ref[k]), k
        fin = dst.finish_codes(d)
        assert _eq({i: fin[d[i]] for i in range(4)}, ref_fin)


@pytest.mark.gpu
def test_move_launch_count_does_not_grow(built_lib):
    import facodec_b200 as fb
    m = _codec()
    x = _wave(3000, 50)
    with fb.CodecStreamPool(m, capacity=40, n_c=2) as src, fb.CodecStreamPool(m, capacity=49, n_c=2) as dst:
        s = [src.open() for _ in range(40)]
        src.encode_codes({i: x for i in s})
        counts = []
        for n in (1, 8, 40):
            states = src.export(s[:n])
            counts.append(_launches(src))
            for i in s[:n][:3]:
                dst.import_session(states[i])
                counts.append(_launches(dst))
        assert len(set(counts)) == 1 and counts[0] == 5, counts
    rs = fb.ResamplePool(capacity=40)
    r = [rs.open(48000, 24000) for _ in range(40)]
    rs.push({i: x[0, 0] for i in r})
    ns = []
    for n in (1, 8, 40):
        rs.export(r[:n])
        ns.append(_launches(rs))
    assert ns == [1, 1, 1]


@pytest.mark.gpu
def test_48k_sessions_move(built_lib):
    """Codes, voice-conversion and decode sessions at 48 kHz carry their resampler sessions (pending input, counters,
    held samples) along; the codes equal Codec.encode of the resampled audio."""
    import facodec_b200 as fb
    m = _codec()
    T = 48000 * 3
    x = _wave(T, 60)
    for at in (1, 3):                              # holding fewer than 3000 samples at 24 kHz; mid-stream
        kind = Kind(lambda p: p.open(sample_rate=48000), lambda p, f: p.encode_codes(f), lambda p, s: p.finish_codes(s),
                    lambda dev="cuda:0": _feeds(T, [2000, 1000, 9000, 4411], lambda q, n: x[:, :, q:q + n].to(dev)))
        src = fb.CodecStreamPool(m, capacity=4, n_c=2)
        dst = fb.CodecStreamPool(_codec(fresh=True), capacity=3, n_c=2)
        a = kind.open(dst)                          # the target already runs a session at 48 kHz
        move_and_compare(kind, src, dst, at, lambda st: fb.SessionState.from_bytes(st.to_bytes()))
        dst.close(a)
    # against Codec.encode: one more moved session, collected
    src = fb.CodecStreamPool(m, capacity=2, n_c=2)
    dst = fb.CodecStreamPool(m, capacity=2, n_c=2)
    s = src.open(sample_rate=48000)
    parts = []
    from test_gpu_stream import chunks_of
    for k, (p, n) in enumerate(chunks_of(T, [2000, 1000, 9000, 4411])):
        if k == 1:
            st = src.export([s])[s]
            assert st.rate is not None and 0 < st.info["held"].numel() < 3000
            src.close(s)
            s, src = dst.import_session(st), dst
        parts.append(src.encode_codes({s: x[:, :, p:p + n]})[s])
    codes, _ = src.finish_codes([s])[s]
    parts.append(codes)
    got = [torch.cat([q[r] for q in parts], dim=2) for r in range(3)]
    r = fb.resample(x, 48000, 24000)
    L = r.shape[2] // 300 * 300
    off, _ = fb.Codec(m).encode(r[:, :, :L], 2)
    assert _eq(got, off)
    g = torch.Generator().manual_seed(23)
    tv = torch.randn(1, 1024, generator=g).cuda()
    vsrc = fb.VoiceConversionPool(_redec(), capacity=4, n_c=1)
    for at in (0, 2, 5):
        move_and_compare(_vc_kind(tv, sample_rate=48000), vsrc, vsrc, at, lambda st: fb.SessionState.from_bytes(st.to_bytes()))
    dsrc = fb.CodecDecodePool(m, capacity=4)
    for at in (0, 2, 5):
        move_and_compare(_dec_kind(tv, sample_rate=48000), dsrc, dsrc, at, lambda st: st)


@pytest.mark.gpu
def test_move_to_second_device(built_lib):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import facodec_b200 as fb
    from facodec_b200 import synth
    sds = synth.synth_state_dicts(0)
    m1 = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        m1[k].load_state_dict(sds[k])
        m1[k].eval()
    src = fb.CodecStreamPool(_codec(), capacity=4, n_c=2)
    dst = fb.CodecStreamPool(m1, capacity=4, n_c=2, device="cuda:1")
    move_and_compare(_codes_kind(), src, dst, 3, lambda st: st)
    g = torch.Generator().manual_seed(24)
    tv = torch.randn(1, 1024, generator=g).cuda()
    dsrc = fb.CodecDecodePool(_codec(), capacity=4)
    ddst = fb.CodecDecodePool(m1, capacity=4, device="cuda:1")
    move_and_compare(_dec_kind(tv), dsrc, ddst, 3, lambda st: st.cpu())


def _header_with(st, **fields):
    """st's state with header fields replaced (the checksum recomputed)."""
    import facodec_b200 as fb
    v = list(HEADER.unpack(st.header))
    names = ["magic", "version", "kind", "header_bytes", "fingerprint"]
    for k, val in fields.items():
        v[names.index(k)] = val
    body = HEADER.pack(*v)[:-8]
    return fb.SessionState(st.kind, body + struct.pack("<Q", fnv1a(body)), st.payload, st.info, st.rate)


@pytest.mark.gpu
def test_rejected_imports_change_nothing(built_lib):
    import facodec_b200 as fb
    m = _codec()
    kind = _codes_kind()
    feeds = kind.feeds()
    src = fb.CodecStreamPool(m, capacity=4, n_c=2)
    dst = fb.CodecStreamPool(m, capacity=3, n_c=2)
    a, t = src.open(), src.open()
    b, u = dst.open(), dst.open()
    for f in feeds[:3]:
        src.encode_codes({a: f, t: f})
        dst.encode_codes({b: f, u: f})
    st = src.export([a])[a]
    bad = []
    flipped = bytearray(st.header)
    flipped[60] ^= 1
    bad.append(fb.SessionState(st.kind, bytes(flipped), st.payload, st.info))           # bit flip
    bad.append(fb.SessionState(st.kind, st.header[:-4], st.payload, st.info))           # truncated header
    bad.append(fb.SessionState(st.kind, st.header, st.payload[:-4], st.info))           # payload shorter than its header
    bad.append(_header_with(st, version=VERSION + 1))                                   # another format version
    bad.append(_header_with(st, fingerprint=HEADER.unpack(st.header)[4] ^ 1))           # other weights
    for s in bad:
        with pytest.raises((fb.FacError, ValueError)):
            dst.import_session(s)
    with pytest.raises(fb.FacError):                                                    # a codes state in a decode pool
        with fb.CodecDecodePool(m, capacity=2) as dp:
            dp._import_state(st)
    with pytest.raises(ValueError):
        with fb.CodecDecodePool(m, capacity=2) as dp:
            dp.import_session(st)
    with fb.CodecStreamPool(_codec(1, fresh=True), capacity=2, n_c=2) as other:         # another synthetic seed
        with pytest.raises(fb.FacError):
            other.import_session(st)
    with fb.CodecStreamPool(m, capacity=2, n_c=1) as other:                             # pool n_c 1 vs 2
        with pytest.raises(fb.FacError):
            other.import_session(st)
    m2 = _codec(fresh=True)                                                             # one option changed
    m2.encoder._engine.set_option("attention_stream", 1, torch.device("cuda:0"))
    with fb.CodecStreamPool(m2, capacity=2, n_c=2) as other:
        with pytest.raises(fb.FacError):
            other.import_session(st)
    with fb.CodecStreamPool(m, capacity=1, n_c=2) as full:                              # a full pool
        full.open()
        with pytest.raises(fb.FacError):
            full.import_session(st)
    e = dst.engine                                                                      # a host payload (C level)
    host = st.payload.cpu()
    hdr = ctypes.create_string_buffer(st.header, len(st.header))
    assert e.L.fac_codes_pool_import(e.handle, dst.pid, hdr, len(st.header), ctypes.c_void_p(host.data_ptr()), host.numel(),
                                     None) == -1
    # export of a finished or closed session
    c = src.open()
    src.encode_codes({c: feeds[0]})
    src.finish_codes([c])
    with pytest.raises(fb.FacError):
        src.export([c])
    src.close(c)
    with pytest.raises(fb.FacError):
        src.export([c])
    # every session of both pools still equals its twin
    for f in feeds[3:]:
        o1 = src.encode_codes({a: f, t: f})
        o2 = dst.encode_codes({b: f, u: f})
        assert _eq(o1[a], o1[t]) and _eq(o2[b], o2[u]) and _eq(o1[a], o2[b])
    assert len(dst._open) == 2 and len(src._open) == 2
    f1, f2 = src.finish_codes([a, t]), dst.finish_codes([b, u])
    assert _eq(f1[a], f1[t]) and _eq(f2[b], f2[u]) and _eq(f1[a], f2[b])
    # a resampler state whose quantum differs, and an export of a finished resampler session
    rs1, rs300 = fb.ResamplePool(capacity=2), fb.ResamplePool(capacity=2, quantum=300)
    r = rs1.open(48000, 24000)
    rs1.push({r: _wave(4000, 70)[0, 0]})
    with pytest.raises(fb.FacError):
        rs300.import_session(rs1.export([r])[r])
    assert not rs300._open
    rs1.finish([r])
    with pytest.raises(fb.FacError):
        rs1.export([r])
