"""Streaming voice conversion through the redecoder (VoiceConversionStream), synthetic checkpoints 0, 20-frame (0.25 s) chunks:

* B = 1, a live pipeline on --utts utterances of --seconds each (30 s: the reference's crop): each 6000-sample chunk of the
  source goes through CodecStream.encode_codes, and its codes through VoiceConversionStream.convert with the timbre of a
  reference clip.  Wall time per chunk of convert alone and of the whole pipeline (encode_codes + convert), host clock around
  a device synchronise, after a warm-up utterance; median and p99.
* B = 32 x 4 s (the bench.py batch, seed 114514): the codes of Codec.encode converted in 20-frame chunks against one
  VoiceConverter.convert on the same codes, alternating, in audio-seconds per second (fastest of --rounds rounds); the
  streamed waveform is checked against the offline one (bit-equal).

    python scripts/stream_vc_bench.py [--rounds 3] [--utts 2] [--seconds 30]

Prints the card, its power limit, its max SM clock and the SM clock sampled right after the timed rounds, then one JSON line.
Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from conv_layer_profile import BATCH, SEED, UTT_SAMPLES, card_info  # noqa: E402

SR, HOP, CHUNK_FRAMES = 24000, 300, 20
CHUNK = CHUNK_FRAMES * HOP


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def sm_clock_mhz(index):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        return float(out.strip())
    except Exception as exc:     # the timings stand without it; say why it is missing
        return f"nvidia-smi: {exc}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="streamed / offline rounds of the B = 32 batch, alternating")
    ap.add_argument("--utts", type=int, default=2, help="B = 1 utterances timed")
    ap.add_argument("--seconds", type=float, default=30.0, help="length of each B = 1 utterance")
    args = ap.parse_args()
    if args.rounds < 1 or args.utts < 1 or args.seconds * SR < 2 * CHUNK:
        ap.error("--rounds and --utts must be >= 1, --seconds >= 0.5")

    import torch
    import facodec_b200 as fb
    from facodec_b200 import synth

    assert torch.cuda.is_available(), "stream_vc_bench.py needs a CUDA device"
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
    converter = fb.VoiceConverter(vc_model)

    # ---- B = 1: the live pipeline, per chunk ----
    T1 = int(args.seconds * SR) // CHUNK * CHUNK
    waves = synth.synth_waves(args.utts + 1, T1, seed=SEED + 1).cuda()
    _, timbre1 = codec.encode(synth.synth_waves(1, 3 * SR, seed=SEED + 2).cuda(), 2)    # the target voice

    def one_utterance(x):
        """Streams one [1,1,T1] utterance; returns the per-chunk wall times (ms) of convert and of the whole pipeline."""
        conv, pipe = [], []
        with fb.CodecStream(codec_model, 1) as tx, fb.VoiceConversionStream(vc_model, 1, timbre1) as vc:
            for p in range(0, T1, CHUNK):
                chunk = x[:, :, p:p + CHUNK].contiguous()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                codes = tx.encode_codes(chunk, 2)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                vc.convert(codes)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                conv.append((t2 - t1) * 1e3)
                pipe.append((t2 - t0) * 1e3)
            vc.convert(tx.finish_codes()[0])
            vc.finish()
        return conv, pipe

    one_utterance(waves[:1])                       # warm-up: sizes the workspaces, loads the modules
    conv_ms, pipe_ms = [], []
    for i in range(1, args.utts + 1):
        c, p = one_utterance(waves[i:i + 1])
        conv_ms += c
        pipe_ms += p

    # ---- B = 32 x 4 s: streamed conversion against VoiceConverter.convert, alternating ----
    x = synth.synth_waves(BATCH, UTT_SAMPLES, seed=SEED).contiguous().cuda()
    codes, timbre = codec.encode(x, 2)
    T = codes[0].shape[-1]

    def streamed():
        with fb.VoiceConversionStream(vc_model, BATCH, timbre) as s:
            ys = [s.convert([codes[0][:, :, p:p + CHUNK_FRAMES], codes[1][:, :, p:p + CHUNK_FRAMES]])
                  for p in range(0, T, CHUNK_FRAMES)]
            ys.append(s.finish())
        return torch.cat(ys, dim=2)

    def offline():
        return converter.convert(codes, timbre)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    for _ in range(2):
        streamed()
        offline()
    ms = {"streamed": [], "offline": []}
    for _ in range(args.rounds):
        ms["streamed"].append(timed(streamed))
        ms["offline"].append(timed(offline))
    clock = sm_clock_mhz(0)
    bit_equal = bool(torch.equal(streamed(), offline()))

    card = card_info(0)
    print(f"card: {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['max_sm_mhz']} MHz, "
          f"SM clock after the B = 32 rounds {clock} MHz" + (f" ({card['error']})" if "error" in card else ""))
    audio_s = BATCH * UTT_SAMPLES / SR
    res = {"card": card, "sm_clock_mhz_after_rounds": clock, "chunk_frames": CHUNK_FRAMES,
           "b1": {"utterances": args.utts, "seconds_each": T1 / SR, "chunks": len(conv_ms),
                  "convert_ms": {"median": round(pct(conv_ms, 0.5), 3), "p99": round(pct(conv_ms, 0.99), 3)},
                  "encode_codes_plus_convert_ms": {"median": round(pct(pipe_ms, 0.5), 3), "p99": round(pct(pipe_ms, 0.99), 3)}},
           "b32": {"workload": f"{BATCH} x {UTT_SAMPLES / SR:g} s utterances, seed {SEED}", "rounds": args.rounds,
                   "streamed_equal_offline": bit_equal}}
    for k, v in ms.items():
        res["b32"][k] = {"ms": [round(t, 2) for t in v], "audio_s_per_s_fastest_round": round(audio_s / (min(v) * 1e-3), 1)}
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
