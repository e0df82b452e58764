"""Streaming compression to codes (CodecStream.encode_codes / finish_codes) and streaming decode from codes (decode_codes),
synthetic checkpoint 0, 0.25 s chunks (6000 samples at 24 kHz):

* B = 1: one sender and one receiver on the same stream; wall time per encode_codes call and per decode_codes call (host
  clock around a device synchronise, after a warm-up utterance), median and p99 over --utts utterances of --seconds each.
* B = 32 x 4 s (the bench.py batch, seed 114514): the batch streamed in 0.25 s chunks against Codec.encode on the same input
  in the same process, alternating, in audio-seconds per second; the streamed codes and timbre are checked against
  Codec.encode's (bit-equal).

    python scripts/stream_codes_bench.py [--rounds 3] [--utts 4] [--seconds 10]

Prints the card, its power limit and max SM clock, then one JSON line.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from conv_layer_profile import BATCH, SEED, UTT_SAMPLES, card_info  # noqa: E402

SR, CHUNK, N_C = 24000, 6000, 2


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="streamed / offline rounds of the B = 32 batch, alternating")
    ap.add_argument("--utts", type=int, default=4, help="B = 1 utterances timed")
    ap.add_argument("--seconds", type=float, default=10.0, help="length of each B = 1 utterance")
    args = ap.parse_args()
    if args.rounds < 1 or args.utts < 1 or args.seconds * SR < CHUNK:
        ap.error("--rounds and --utts must be >= 1, --seconds >= 0.25")

    import torch
    import facodec_b200 as fb
    from facodec_b200 import synth

    assert torch.cuda.is_available(), "stream_codes_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    sds = synth.synth_state_dicts(0)
    model = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        model[k].load_state_dict(sds[k])
        model[k].eval()
    codec = fb.Codec(model)

    # ---- B = 1: per-call latency of a sender (encode_codes) and a receiver (decode_codes) ----
    T1 = int(args.seconds * SR) // CHUNK * CHUNK
    waves = synth.synth_waves(args.utts + 1, T1, seed=SEED + 1).cuda()

    def one_utterance(x):
        """Streams one [1,1,T1] utterance; returns the per-call wall times (ms) of encode_codes and decode_codes."""
        _, timbre = codec.encode(x, N_C)          # the receiver's voice: any timbre will do
        enc, dec = [], []
        with fb.CodecStream(model, 1) as s:
            for p in range(0, T1, CHUNK):
                chunk = x[:, :, p:p + CHUNK].contiguous()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                codes = s.encode_codes(chunk, N_C)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                s.decode_codes(codes, timbre)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                enc.append((t1 - t0) * 1e3)
                dec.append((t2 - t1) * 1e3)
            s.decode_codes(s.finish_codes()[0], timbre)
        return enc, dec

    one_utterance(waves[:1])                       # warm-up: sizes the workspace, loads the modules
    enc_ms, dec_ms = [], []
    for i in range(1, args.utts + 1):
        e, d = one_utterance(waves[i:i + 1])
        enc_ms += e
        dec_ms += d

    # ---- B = 32 x 4 s: streamed compression against Codec.encode, alternating ----
    x = synth.synth_waves(BATCH, UTT_SAMPLES, seed=SEED).contiguous().cuda()

    def streamed():
        with fb.CodecStream(model, BATCH) as s:
            parts = [s.encode_codes(x[:, :, p:p + CHUNK].contiguous(), N_C) for p in range(0, UTT_SAMPLES, CHUNK)]
            last, timbre = s.finish_codes()
        return [torch.cat([q[i] for q in parts] + [last[i]], dim=2) for i in range(3)], timbre

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    for _ in range(2):
        streamed()
        codec.encode(x, N_C)
    ms = {"streamed": [], "offline": []}
    for _ in range(args.rounds):
        ms["streamed"].append(timed(streamed)[0])
        ms["offline"].append(timed(lambda: codec.encode(x, N_C))[0])
    (codes_st, timbre_st), (codes_off, timbre_off) = streamed(), codec.encode(x, N_C)
    bit_equal = all(torch.equal(a, b) for a, b in zip(codes_st, codes_off)) and torch.equal(timbre_st, timbre_off)

    card = card_info(0)
    print(f"card: {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['max_sm_mhz']} MHz"
          + (f" ({card['error']})" if "error" in card else ""))
    audio_s = BATCH * UTT_SAMPLES / SR
    res = {"card": card, "chunk_samples": CHUNK, "n_c": N_C,
           "b1": {"utterances": args.utts, "seconds_each": T1 / SR, "calls": len(enc_ms),
                  "encode_codes_ms": {"median": round(pct(enc_ms, 0.5), 3), "p99": round(pct(enc_ms, 0.99), 3)},
                  "decode_codes_ms": {"median": round(pct(dec_ms, 0.5), 3), "p99": round(pct(dec_ms, 0.99), 3)}},
           "b32": {"workload": f"{BATCH} x {UTT_SAMPLES / SR:g} s utterances, seed {SEED}", "rounds": args.rounds,
                   "streamed_codes_equal_offline": bit_equal}}
    for k, v in ms.items():
        res["b32"][k] = {"ms": [round(t, 2) for t in v], "audio_s_per_s_fastest_round": round(audio_s / (min(v) * 1e-3), 1)}
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
