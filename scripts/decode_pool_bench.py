"""Codec receivers for S live sessions at once (CodecDecodePool): codes in, audio out, synthetic checkpoint 0.  Every receiver
gets --chunks chunks whose lengths are drawn from 15-25 frames (fixed seed; the sender or the network chooses them), starts
at step i % 8 (staggered joins and leaves) and decodes with its own timbre; every 4th receiver switches between 3 and 1
residual rows (its bitrate) from step to step.

* pool: one step = one decode_codes over the current receivers.  Wall time per step, host clock around a device
  synchronise: median and p99, the real-time capacity S x mean chunk duration / median step time, and the batches per step
  of the launch plan (fac_debug_pool_plan kind 2).
* b1: S B = 1 CodecStream.decode_codes stepped one after another over the same schedule, per step.
* lockstep: the same number of receivers in ceil(S / 32) B = 32 streams fed uniform 20-frame chunks together (every row
  starts and ends at once): an upper bound, not a way to serve receivers whose chunk lengths differ.
The three alternate in the same process (--rounds rounds each); every receiver's pool output is checked against its B = 1
output (bit-equal).  S in --receivers (default 8, 32, 64, 128).

    python scripts/decode_pool_bench.py [--rounds 2] [--chunks 16] [--receivers 8,32,64,128]

Prints the card, its power limit, its max SM clock and the SM clock sampled right after the timed rounds, then one JSON line.
Needs a CUDA device.
"""
import argparse
import ctypes
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from conv_layer_profile import SEED, card_info  # noqa: E402
from stream_vc_bench import pct, sm_clock_mhz  # noqa: E402

SR, HOP, LOCKSTEP_FRAMES = 24000, 300, 20
FRAME_MS = HOP * 1e3 / SR


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2, help="rounds of each of pool / b1 / lockstep, alternating")
    ap.add_argument("--chunks", type=int, default=16, help="chunks per receiver (16 x ~20 frames ~ 4 s)")
    ap.add_argument("--receivers", default="8,32,64,128", help="comma-separated S")
    args = ap.parse_args()
    receivers = [int(s) for s in args.receivers.split(",")]
    if args.rounds < 1 or args.chunks < 1 or min(receivers) < 1:
        ap.error("--rounds >= 1, --chunks >= 1, receivers >= 1")

    import numpy as np
    import torch
    import facodec_b200 as fb
    from facodec_b200 import synth

    assert torch.cuda.is_available(), "decode_pool_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    sds = synth.synth_state_dicts(0)
    model = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        model[k].load_state_dict(sds[k])
        model[k].eval()
    L = model.decoder._engine.L

    smax = max(receivers)
    rng = random.Random(SEED)
    lens = [[rng.randint(15, 25) for _ in range(args.chunks)] for _ in range(smax)]
    rows = [[(2, 3 if i % 4 != 3 or k % 2 == 0 else 1) for k in range(args.chunks)] for i in range(smax)]
    g = torch.Generator().manual_seed(SEED + 5)
    Tmax = max(max(sum(x) for x in lens), args.chunks * LOCKSTEP_FRAMES)     # lockstep reads 20 frames per chunk
    codes = [torch.randint(0, 1024, (smax, r, Tmax), generator=g).cuda() for r in (1, 2, 3)]
    _, timbres = fb.Codec(model).encode(synth.synth_waves(smax, 3 * SR, seed=SEED + 4).cuda(), 2)   # one voice per receiver
    starts = [[sum(x[:k]) for k in range(args.chunks)] for x in lens]

    def chunk(i, k):
        p, F = starts[i][k], lens[i][k]
        nc, nr = rows[i][k]
        return [codes[0][i:i + 1, :, p:p + F], codes[1][i:i + 1, :nc, p:p + F], codes[2][i:i + 1, :nr, p:p + F]]

    def sync_ms(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    def schedule(S):
        """Per step, the receivers feeding chunk k: receiver i feeds chunk step - i % 8."""
        return [[(i, step - i % 8) for i in range(S) if 0 <= step - i % 8 < args.chunks] for step in range(args.chunks + 7)]

    def plan_batches(feed):
        frames = np.array([starts[i][k] for i, k in feed], dtype=np.int64)
        ln = np.array([lens[i][k] for i, k in feed], dtype=np.int32)
        grp, bat = np.zeros(len(feed), dtype=np.int32), np.zeros(len(feed), dtype=np.int32)
        P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        return L.fac_debug_pool_plan(2, len(feed), P(frames), P(ln), P(grp), P(bat))

    def run_pool(S):
        ys, times = [[] for _ in range(S)], []
        with fb.CodecDecodePool(model, capacity=S) as pool:
            sid = {}

            def step(feed):
                for i, k in feed:
                    if k == 0:
                        sid[i] = pool.open(timbres[i:i + 1])
                out = pool.decode_codes({sid[i]: chunk(i, k) for i, k in feed})
                for i, k in feed:
                    ys[i].append(out[sid[i]])
                    if k == args.chunks - 1:
                        pool.close(sid[i])

            for feed in schedule(S):
                times.append(sync_ms(lambda: step(feed)))
        return [torch.cat(y, dim=2) for y in ys], times

    def run_b1(S):
        ys, times, streams = [[] for _ in range(S)], [], {}

        def step(feed):
            for i, k in feed:
                if k == 0:
                    streams[i] = fb.CodecStream(model, 1)
                ys[i].append(streams[i].decode_codes(chunk(i, k), timbres[i:i + 1]))
                if k == args.chunks - 1:
                    streams[i].close()

        for feed in schedule(S):
            times.append(sync_ms(lambda: step(feed)))
        return [torch.cat(y, dim=2) for y in ys], times

    def run_lockstep(S):
        times = []
        groups = (S + 31) // 32
        for b0 in range(0, S, 32):
            B = min(32, S - b0)
            with fb.CodecStream(model, B) as st:
                for k in range(args.chunks):
                    p = k * LOCKSTEP_FRAMES
                    c = [codes[0][b0:b0 + B, :, p:p + LOCKSTEP_FRAMES], codes[1][b0:b0 + B, :, p:p + LOCKSTEP_FRAMES],
                         codes[2][b0:b0 + B, :, p:p + LOCKSTEP_FRAMES]]
                    times.append(sync_ms(lambda: st.decode_codes(c, timbres[b0:b0 + B])))
        # per step of the pool's meaning: all ceil(S/32) groups advance one chunk
        return [sum(times[gi * args.chunks + k] for gi in range(groups)) for k in range(args.chunks)]

    run_pool(min(receivers))                       # warm-up: sizes the workspaces, loads the modules
    run_b1(1)
    run_lockstep(1)
    mean_chunk_ms = float(np.mean(lens)) * FRAME_MS
    res = {"mean_chunk_ms": round(mean_chunk_ms, 2), "lockstep_chunk_ms": LOCKSTEP_FRAMES * FRAME_MS, "chunks_each": args.chunks,
           "rounds": args.rounds, "receivers": {}}
    for S in receivers:
        ms = {"pool": [], "b1": [], "lockstep": []}
        equal = True
        for _ in range(args.rounds):
            yp, tp = run_pool(S)
            yb, tb = run_b1(S)
            tl = run_lockstep(S)
            equal &= all(torch.equal(a, b) for a, b in zip(yp, yb))
            ms["pool"] += tp
            ms["b1"] += tb
            ms["lockstep"] += tl
        nb = [plan_batches(feed) for feed in schedule(S)]
        r = {"pool_equal_b1": equal, "pool_batches_per_step_median": float(np.median(nb)), "pool_batches_per_step_max": int(max(nb))}
        for k, v in ms.items():
            med = pct(v, 0.5)
            chunk_ms = LOCKSTEP_FRAMES * FRAME_MS if k == "lockstep" else mean_chunk_ms
            r[k] = {"step_ms_median": round(med, 3), "step_ms_p99": round(pct(v, 0.99), 3),
                    "realtime_receivers": round(S * chunk_ms / med, 1)}
        res["receivers"][S] = r
    clock = sm_clock_mhz(0)
    card = card_info(0)
    print(f"card: {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['max_sm_mhz']} MHz, "
          f"SM clock after the timed rounds {clock} MHz" + (f" ({card['error']})" if "error" in card else ""))
    res["card"], res["sm_clock_mhz_after_rounds"] = card, clock
    print(json.dumps(res))
    return 0 if all(r["pool_equal_b1"] for r in res["receivers"].values()) else 1


if __name__ == "__main__":
    sys.exit(main())
