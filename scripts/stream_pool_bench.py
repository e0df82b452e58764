"""Live voice conversion for S callers at once (CodecStreamPool -> VoiceConversionPool), synthetic checkpoints 0, 0.25 s
(6000-sample, 20-frame) chunks, every caller a --seconds utterance starting at step i % 8 (staggered joins and leaves):

* pool: one step = encode_codes over the current callers, then convert of their codes (and the finishes of the callers whose
  utterance ended).  Wall time per step, host clock around a device synchronise: median and p99, and the real-time capacity
  S x 250 ms / median step time.
* b1: S B = 1 CodecStream + VoiceConversionStream pairs stepped one after another over the same schedule, per step.
* lockstep: the same audio in ceil(S / 32) B = 32 stream pairs stepped together (every row starts and ends at once).
The three alternate in the same process (--rounds rounds each); every caller's pool output is checked against its B = 1
output (bit-equal).  S in --callers (default 8, 32, 64, 128).

    python scripts/stream_pool_bench.py [--rounds 2] [--seconds 4] [--callers 8,32,64,128]

Prints the card, its power limit, its max SM clock and the SM clock sampled right after the timed rounds, then one JSON line.
Needs a CUDA device.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from conv_layer_profile import SEED, card_info  # noqa: E402
from stream_vc_bench import pct, sm_clock_mhz  # noqa: E402

SR, HOP, CHUNK_FRAMES = 24000, 300, 20
CHUNK = CHUNK_FRAMES * HOP


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2, help="rounds of each of pool / b1 / lockstep, alternating")
    ap.add_argument("--seconds", type=float, default=4.0, help="length of every caller's utterance")
    ap.add_argument("--callers", default="8,32,64,128", help="comma-separated S")
    args = ap.parse_args()
    callers = [int(s) for s in args.callers.split(",")]
    if args.rounds < 1 or args.seconds * SR < 2 * CHUNK or min(callers) < 1:
        ap.error("--rounds >= 1, --seconds >= 0.5, callers >= 1")

    import torch
    import facodec_b200 as fb
    from facodec_b200 import synth

    assert torch.cuda.is_available(), "stream_pool_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    sds = synth.synth_state_dicts(0)
    codec_model = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        codec_model[k].load_state_dict(sds[k])
        codec_model[k].eval()
    rsds = synth.synth_redecoder_state_dicts(0)
    vc_model = fb.build_model(stage="redecoder")
    for k in ("encoder", "decoder"):
        vc_model[k].load_state_dict(rsds[k])
        vc_model[k].eval()
    codec = fb.Codec(codec_model)

    T = int(args.seconds * SR) // CHUNK * CHUNK
    nchunks = T // CHUNK
    smax = max(callers)
    waves = synth.synth_waves(smax, T, seed=SEED + 3).cuda()
    _, timbres = codec.encode(synth.synth_waves(smax, 3 * SR, seed=SEED + 4).cuda(), 2)   # one target voice per caller

    def sync_ms(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    def schedule(S):
        """Per step, the callers feeding chunk k: caller i feeds chunk step - i % 8."""
        return [[(i, step - i % 8) for i in range(S) if 0 <= step - i % 8 < nchunks] for step in range(nchunks + 7)]

    def run_pool(S):
        ys, times = [[] for _ in range(S)], []
        with fb.CodecStreamPool(codec_model, capacity=S, n_c=2) as tx, fb.VoiceConversionPool(vc_model, capacity=S, n_c=1) as vc:
            cs, vs = {}, {}

            def step(feed):
                for i, k in feed:
                    if k == 0:
                        cs[i], vs[i] = tx.open(), vc.open(timbres[i:i + 1])
                codes = tx.encode_codes({cs[i]: waves[i:i + 1, :, k * CHUNK:(k + 1) * CHUNK] for i, k in feed})
                out = vc.convert({vs[i]: codes[cs[i]] for i, _ in feed})
                for i, _ in feed:
                    ys[i].append(out[vs[i]])
                ending = [i for i, k in feed if k == nchunks - 1]
                if ending:
                    fin = tx.finish_codes([cs[i] for i in ending])
                    out = vc.convert({vs[i]: fin[cs[i]][0] for i in ending})
                    tail = vc.finish([vs[i] for i in ending])
                    for i in ending:
                        ys[i] += [out[vs[i]], tail[vs[i]]]
                        tx.close(cs[i])
                        vc.close(vs[i])

            for feed in schedule(S):
                times.append(sync_ms(lambda: step(feed)))
        return [torch.cat(y, dim=2) for y in ys], times

    def run_b1(S):
        ys, times = [[] for _ in range(S)], []
        pairs = {}

        def step(feed):
            for i, k in feed:
                if k == 0:
                    pairs[i] = (fb.CodecStream(codec_model, 1), fb.VoiceConversionStream(vc_model, 1, timbres[i:i + 1]))
                tx, vc = pairs[i]
                ys[i].append(vc.convert(tx.encode_codes(waves[i:i + 1, :, k * CHUNK:(k + 1) * CHUNK].contiguous(), 2)))
                if k == nchunks - 1:
                    ys[i] += [vc.convert(tx.finish_codes()[0]), vc.finish()]
                    tx.close()
                    vc.close()

        for feed in schedule(S):
            times.append(sync_ms(lambda: step(feed)))
        return [torch.cat(y, dim=2) for y in ys], times

    def run_lockstep(S):
        times = []
        for b0 in range(0, S, 32):
            B = min(32, S - b0)
            with fb.CodecStream(codec_model, B) as tx, fb.VoiceConversionStream(vc_model, B, timbres[b0:b0 + B]) as vc:
                for k in range(nchunks):
                    times.append(sync_ms(lambda: vc.convert(tx.encode_codes(waves[b0:b0 + B, :, k * CHUNK:(k + 1) * CHUNK]
                                                                            .contiguous(), 2))))
                vc.convert(tx.finish_codes()[0])
                vc.finish()
        # per step of the pool's meaning: all ceil(S/32) groups advance one chunk
        groups = (S + 31) // 32
        return [sum(times[g * nchunks + k] for g in range(groups)) for k in range(nchunks)]

    run_pool(min(callers))                    # warm-up: sizes the workspaces, loads the modules
    run_b1(1)
    run_lockstep(1)
    res = {"chunk_ms": CHUNK * 1e3 / SR, "seconds_each": T / SR, "rounds": args.rounds, "callers": {}}
    for S in callers:
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
        r = {"pool_equal_b1": equal}
        for k, v in ms.items():
            med = pct(v, 0.5)
            r[k] = {"step_ms_median": round(med, 3), "step_ms_p99": round(pct(v, 0.99), 3),
                    "realtime_callers": round(S * CHUNK * 1e3 / SR / med, 1)}
        res["callers"][S] = r
    clock = sm_clock_mhz(0)
    card = card_info(0)
    print(f"card: {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['max_sm_mhz']} MHz, "
          f"SM clock after the timed rounds {clock} MHz" + (f" ({card['error']})" if "error" in card else ""))
    res["card"], res["sm_clock_mhz_after_rounds"] = card, clock
    print(json.dumps(res))
    return 0 if all(r["pool_equal_b1"] for r in res["callers"].values()) else 1


if __name__ == "__main__":
    sys.exit(main())
