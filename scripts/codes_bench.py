"""Compress-only and decompress throughput at the bench.py workload (32 x 4 s utterances, seed 114514, synthetic checkpoint 0):
Codec.forward, Codec.encode and Codec.decode timed in the same process, alternating, with CUDA events after warm-up.

    python scripts/codes_bench.py [--steps 10] [--rounds 3] [--warmup 3]

Prints the card, its power limit and max SM clock, then one JSON line: ms per step and audio-seconds per second of each
call, the B = 1 decode latency (one 4 s utterance), the "dequantize" kernel family's device time per step and achieved
GB/s from the library's launch profiler (a separate profiled pass: events around every launch slow the host, so the
step times above come from the unprofiled passes), and the RMS of decode(*encode(x)) against forward(x) on the timed
batch.  Needs a CUDA device.
"""
import argparse
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from conv_layer_profile import BATCH, SEED, UTT_SAMPLES, card_info  # noqa: E402

UTT_SECONDS = UTT_SAMPLES / 24000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed calls of each kind per round")
    ap.add_argument("--rounds", type=int, default=3, help="forward / encode / decode rounds, alternating")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1 or args.rounds < 1:
        ap.error("--steps and --rounds must be >= 1")

    import torch
    import facodec_b200 as fb
    from facodec_b200 import synth

    assert torch.cuda.is_available(), "codes_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    sds = synth.synth_state_dicts(0)
    model = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        model[k].load_state_dict(sds[k])
        model[k].eval()
    codec = fb.Codec(model)
    x = synth.synth_waves(BATCH, UTT_SAMPLES, seed=SEED).contiguous().cuda()
    codes, timbre = codec.encode(x)
    calls = {"forward": lambda: codec.forward(x), "encode": lambda: codec.encode(x), "decode": lambda: codec.decode(codes, timbre)}

    def timed(fn, steps):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / steps

    for fn in calls.values():
        for _ in range(args.warmup):
            fn()
    ms = {k: [] for k in calls}
    for _ in range(args.rounds):
        for k, fn in calls.items():
            ms[k].append(timed(fn, args.steps))

    # B = 1 decode latency: one utterance's codes, synchronised per call
    codes1 = [c[:1].contiguous() for c in codes]
    timbre1 = timbre[:1].contiguous()
    for _ in range(args.warmup):
        codec.decode(codes1, timbre1)
    lat = sorted(timed(lambda: codec.decode(codes1, timbre1), 1) for _ in range(max(20, args.steps)))

    # agreement on the timed batch
    y_fwd = codec.forward(x)[0]
    y_dec = codec.decode(*codec.encode(x))
    rms = float(((y_dec.double() - y_fwd.double()) ** 2).mean().sqrt())

    # dequantize kernel family, profiled pass
    L, h = codec.engine.L, codec.engine.handle
    L.fac_profile_reset(h)
    L.fac_profile_enable(h, 1)
    for _ in range(args.steps):
        codec.decode(codes, timbre)
    torch.cuda.synchronize()
    L.fac_profile_enable(h, 0)
    pm, pf, pb, pl = ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong()
    L.fac_profile_get(h, b"dequantize", ctypes.byref(pm), ctypes.byref(pf), ctypes.byref(pb), ctypes.byref(pl))
    L.fac_profile_reset(h)
    deq_ms = pm.value / args.steps

    card = card_info(0)
    print(f"card: {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['max_sm_mhz']} MHz"
          + (f" ({card['error']})" if "error" in card else ""))
    audio_s = BATCH * UTT_SECONDS
    res = {"workload": f"{BATCH} x {UTT_SECONDS:g} s utterances, n_c = 2, seed {SEED}, synthetic checkpoint 0",
           "card": card, "steps": args.steps, "rounds": args.rounds}
    for k, v in ms.items():
        best = min(v)
        res[k] = {"ms_per_step": [round(t, 3) for t in v], "audio_s_per_s_fastest_round": round(audio_s / (best * 1e-3), 1)}
    res["decode_b1_latency_ms"] = {"median": round(lat[len(lat) // 2], 3), "min": round(lat[0], 3)}
    res["dequantize"] = {"ms_per_step": round(deq_ms, 4), "launches_per_step": pl.value // args.steps,
                         "gb_per_s": round(pb.value / (pm.value * 1e-3) / 1e9, 1) if pm.value > 0 else None,
                         "share_of_decode_step": round(deq_ms / min(ms["decode"]), 4)}
    res["decode_of_encode_vs_forward_y_rms"] = rms
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
