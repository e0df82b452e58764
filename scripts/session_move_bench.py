"""Cost of moving live pool sessions: export + import of S sessions, and the first pool step after the move.

For each pool kind (codes, vc, dec, rs) S = 128 sessions are fed 3 s and then 60 s of audio (or its codes).  At each point
the first S = 32 and then all 128 are exported and imported into a second pool (same device; and a pool of a second
engine on cuda:1 when there is one), timed with a device synchronise at the end (fastest of --reps).  The imported
sessions' next step is timed against the same step of the sessions that never moved.  Prints one JSON line per row, then
the card, its power limit and max SM clock (all of it also written to --out when given).

    python scripts/session_move_bench.py [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import facodec_b200 as fb  # noqa: E402
from facodec_b200 import synth  # noqa: E402


def codec_model():
    sds = synth.synth_state_dicts(0)
    m = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        m[k].load_state_dict(sds[k])
        m[k].eval()
    return m


def redec_model():
    sds = synth.synth_redecoder_state_dicts(0)
    m = fb.build_model(stage="redecoder")
    for k in ("encoder", "decoder"):
        m[k].load_state_dict(sds[k])
        m[k].eval()
    return m


def vc_pool(model, device, cap):
    with torch.cuda.device(device):                      # the pool takes its device from the current one
        return fb.VoiceConversionPool(model, capacity=cap, n_c=1)


def timed(fn, device):
    torch.cuda.synchronize(device)
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize(device)
    return time.perf_counter() - t, out


class Setup:
    """A pool kind: make(device) -> pool, open(pool) -> session, feed(seconds, device) -> one session's input for that
    much audio, step(pool, {s: input})."""

    def __init__(self, make, open_fn, feed, step):
        self.make, self.open, self.feed, self.step = make, open_fn, feed, step


def setups(dev1):
    codec0 = codec_model()
    codec1 = codec_model() if dev1 else None
    red0 = redec_model()
    red1 = redec_model() if dev1 else None
    g = torch.Generator().manual_seed(1)
    tv = torch.randn(1, 1024, generator=g)
    wave = synth.synth_waves(1, 24000 * 3, seed=5)
    codes = [torch.randint(0, 1024, (1, r, 240), generator=g) for r in (1, 2, 3)]
    pick = lambda d: (codec0 if str(d) == "cuda:0" else codec1)
    return {
        "codes": Setup(lambda d, cap: fb.CodecStreamPool(pick(d), capacity=cap, n_c=2, device=d), lambda p: p.open(),
                       lambda sec, d: wave[:, :, :24000 * sec].to(d), lambda p, f: p.encode_codes(f)),
        "vc": Setup(lambda d, cap: vc_pool(red0 if str(d) == "cuda:0" else red1, d, cap),
                    lambda p: p.open(tv.to(p.device)), lambda sec, d: [c[:, :, :80 * sec].to(d) for c in codes[:2]],
                    lambda p, f: p.convert(f)),
        "dec": Setup(lambda d, cap: fb.CodecDecodePool(pick(d), capacity=cap, device=d), lambda p: p.open(tv.to(p.device)),
                     lambda sec, d: [c[:, :, :80 * sec].to(d) for c in codes], lambda p, f: p.decode_codes(f)),
        "rs": Setup(lambda d, cap: fb.ResamplePool(capacity=cap, device=d), lambda p: p.open(48000, 24000),
                    lambda sec, d: synth.synth_waves(1, 48000 * sec, seed=6)[0, 0].to(d), lambda p, f: p.push(f)),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sessions", type=int, nargs="+", default=[32, 128])
    ap.add_argument("--kinds", nargs="+", default=["codes", "vc", "dec", "rs"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    torch.cuda.set_device(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    dev1 = "cuda:1" if torch.cuda.device_count() > 1 else None
    S = max(a.sessions)
    rows = []
    for name, k in setups(dev1).items():
        if name not in a.kinds:
            continue
        src = k.make("cuda:0", S)
        sess = [k.open(src) for _ in range(S)]
        fed = 0
        for point in (3, 60):
            while fed < point:                               # 3 s chunks, all sessions in lockstep
                f = k.feed(3, "cuda:0")
                k.step(src, {s: f for s in sess})
                fed += 3
            for n in a.sessions:
                nxt = k.feed(1, "cuda:0")
                for target in ["cuda:0"] + ([dev1] if dev1 else []):
                    dst = k.make(target, n)
                    best, moved = None, None
                    for _ in range(a.reps):
                        if moved:
                            for s in moved:
                                dst.close(s)

                        def move():
                            states = src.export(sess[:n])
                            return [dst.import_session(states[s]) for s in sess[:n]]
                        t, moved = timed(move, target)
                        best = t if best is None else min(best, t)
                    nbytes = sum(st.nbytes for st in src.export(sess[:n]).values())
                    # the moved sessions' next step (fastest of --reps, each on a fresh import) against the same step of
                    # the sessions that never moved (once: it advances them, and the rest follow untimed to stay in step)
                    f_t = [x.to(target) for x in nxt] if isinstance(nxt, list) else nxt.to(target)
                    t_moved = None
                    for _ in range(a.reps):
                        for s in moved:
                            dst.close(s)
                        states = src.export(sess[:n])
                        moved = [dst.import_session(states[s]) for s in sess[:n]]
                        tm, _ = timed(lambda: k.step(dst, {s: f_t for s in moved}), target)
                        t_moved = tm if t_moved is None else min(t_moved, tm)
                    t_native, _ = timed(lambda: k.step(src, {s: nxt for s in sess[:n]}), "cuda:0")
                    if n < S:
                        k.step(src, {s: nxt for s in sess[n:]})
                    fed += 1
                    row = dict(kind=name, audio_s=fed - 1, sessions=n, target=target, move_ms=round(best * 1e3, 3),
                               state_mb=round(nbytes / 2**20, 3), first_step_moved_ms=round(t_moved * 1e3, 3),
                               first_step_native_ms=round(t_native * 1e3, 3))
                    print(json.dumps(row), flush=True)
                    rows.append(row)
                    dst.close()
        src.close()
    print(json.dumps(dict(card=card)))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
