"""The timbre on its own (Codec.timbre, CodecStreamPool.timbre) against what it used to take (Codec.encode):

* offline: Codec.timbre against Codec.encode(n_c = 2) on --batch x --seconds of audio, in --rounds alternating rounds of
  --reps calls each (CUDA events, ms per call; the fastest round counts), and the launches of each call.
* pool: CodecStreamPool.timbre over all S sessions (S in --sessions) once every session has been fed 3 s and again after
  --long seconds (fed in 2 s chunks in between): ms per call (CUDA events over --reps calls, the fastest of --rounds),
  the launches of one call and the number of StyleEncoder batches it plans.

    python scripts/timbre_bench.py [--batch 32] [--seconds 4] [--rounds 5] [--reps 10] [--sessions 32,128] [--long 60]
    python scripts/timbre_bench.py --rehearse      # no GPU: argument parsing and the pool's batch plans

Prints the card, its power limit and max SM clock, then one JSON line (also written to --out when given).  Synthetic
checkpoints (seed 0).
"""
import argparse
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

HOP = 300


def pool_batches(frames):
    """The number of StyleEncoder batches fac_codes_pool_timbre plans for sessions of `frames` mel frames (host only)."""
    from facodec_b200 import _lib
    n = len(frames)
    batch = (ctypes.c_int * max(n, 1))()
    return _lib.load().fac_debug_timbre_plan(n, (ctypes.c_int * max(n, 1))(*frames), batch)


def rehearse(args):
    plans = {}
    for S in args.sessions:
        for sec in (3, args.long):
            plans["S=%d,%gs" % (S, sec)] = pool_batches([int(sec * 24000) // HOP] * S)
    print(json.dumps({"rehearsal": "no GPU: batch plans only", "pool_batches": plans}))


def events_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def model(fb):
    from facodec_b200 import synth
    m = fb.build_model()
    sds = synth.synth_state_dicts(0)
    for k in ("encoder", "quantizer", "decoder"):
        m[k].load_state_dict(sds[k])
        m[k].eval()
    return m


def bench_offline(args, fb, m):
    from facodec_b200 import synth
    codec = fb.Codec(m)
    x = synth.synth_waves(args.batch, int(args.seconds * 24000), seed=5).cuda()
    t = codec.timbre(x)
    n_timbre = codec.launch_count()
    _, ref = codec.encode(x, 2)
    n_encode = codec.launch_count()
    torch.cuda.synchronize()
    assert torch.equal(t, ref), "Codec.timbre differs from Codec.encode's timbre"
    tt, te = [], []
    for _ in range(args.rounds):
        tt.append(events_ms(lambda: codec.timbre(x), args.reps))
        te.append(events_ms(lambda: codec.encode(x, 2), args.reps))
    return {"batch": args.batch, "seconds": args.seconds, "timbre_ms": min(tt), "encode_ms": min(te),
            "timbre_ms_rounds": tt, "encode_ms_rounds": te, "launches_timbre": n_timbre, "launches_encode": n_encode}


def bench_pool(args, fb, m, S):
    from facodec_b200 import synth
    pool = fb.CodecStreamPool(m, capacity=S, n_c=2)
    ss = [pool.open() for _ in range(S)]
    long_T = int(args.long * 24000) // 6000 * 6000
    x = synth.synth_waves(S, max(long_T, 72000), seed=7).cuda()
    out, fed = {}, 0
    for target in (72000, long_T):
        while fed < target:
            n = 72000 if fed == 0 else min(48000, target - fed)
            pool.encode_codes({s: x[i:i + 1, :, fed:fed + n] for i, s in enumerate(ss)})
            fed += n
        pool.timbre(ss)                                   # warm-up: sizes the workspace
        launches = fb.Codec(m).launch_count()
        torch.cuda.synchronize()
        ms = min(events_ms(lambda: pool.timbre(ss), args.reps) for _ in range(args.rounds))
        out["%gs" % (fed / 24000)] = {"ms": ms, "launches": launches, "batches": pool_batches([fed // HOP] * S)}
    pool.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=4.0)
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds; the fastest counts")
    ap.add_argument("--reps", type=int, default=10, help="calls per timed round")
    ap.add_argument("--sessions", default="32,128", help="comma-separated CodecStreamPool sizes")
    ap.add_argument("--long", type=float, default=60.0, help="seconds per session at the second pool measurement")
    ap.add_argument("--rehearse", action="store_true", help="no GPU: the pool's batch plans only")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    args.sessions = [int(s) for s in args.sessions.split(",") if s]
    if args.rounds < 1 or args.reps < 1 or args.batch < 1 or args.seconds <= 0 or args.long < 5 or not args.sessions:
        ap.error("rounds, reps, batch >= 1, seconds > 0, long >= 5, at least one pool size")
    if args.rehearse:
        return rehearse(args)
    if not torch.cuda.is_available():
        sys.exit("timbre_bench.py needs a CUDA device (--rehearse runs the host part)")
    import facodec_b200 as fb
    from conv_layer_profile import card_info
    card = card_info(0)
    print("card:", card)
    m = model(fb)
    out = {"card": card, "offline": bench_offline(args, fb, m),
           "pool": {str(S): bench_pool(args, fb, m, S) for S in args.sessions}}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
