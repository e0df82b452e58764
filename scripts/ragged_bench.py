"""Offline work on a corpus whose utterances all differ in length: Codec.encode / forward (lengths=), Codec.decode and
VoiceConverter.convert (frames=) on ragged batches against one B = 1 call per utterance, synthetic checkpoint 0.

The corpus is --utts utterances with sample counts drawn uniformly from 1-12 s at 24 kHz (any sample count; fixed seed):
synthetic waves for encode / forward, and for decode / convert F = samples // 300 frames of random codes (2 content,
3 residual rows) with a random timbre per utterance.
Three ways to run it, in alternating rounds (--rounds), the fastest round of each reported:
* b1: one call per utterance, one after another;
* arrival: ragged batches of --batch utterances in corpus order, each padded to its longest member;
* sorted: the same after sorting the corpus by length, so a batch's members are close in length.
Each timing is a host clock around the whole corpus, ending in a device synchronise.  Reported in audio-s/s (corpus
seconds over wall seconds), with the padding fraction of each batched order (padded frames / computed frames).  Inside the
run, a sample of lanes of each batched order is checked against its B = 1 output, bit for bit.

    python scripts/ragged_bench.py [--utts 256] [--batch 32] [--rounds 3]

Prints the card, its power limit, its max SM clock and the SM clock sampled right after the timed rounds, then one JSON
line.  Needs a CUDA device.
"""
import argparse
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from conv_layer_profile import SEED, card_info  # noqa: E402
from stream_vc_bench import sm_clock_mhz  # noqa: E402

SR, HOP = 24000, 300


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3, help="rounds of each of b1 / arrival / sorted, alternating")
    ap.add_argument("--check", type=int, default=8, help="lanes per batched order checked against their B = 1 output")
    args = ap.parse_args()
    if args.utts < 1 or args.batch < 1 or args.rounds < 1:
        ap.error("--utts, --batch and --rounds must be >= 1")

    import torch
    import facodec_b200 as fb
    from facodec_b200 import synth

    assert torch.cuda.is_available(), "ragged_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    sds = synth.synth_state_dicts(0)
    model = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        model[k].load_state_dict(sds[k])
        model[k].eval()
    red = fb.build_model(stage="redecoder")
    rsd = synth.synth_redecoder_state_dicts(0)
    for k in ("encoder", "decoder"):
        red[k].load_state_dict(rsd[k])
        red[k].eval()
    codec, vc = fb.Codec(model), fb.VoiceConverter(red)

    rng = random.Random(SEED)
    samples = [rng.randint(1 * SR, 12 * SR) for _ in range(args.utts)]
    frames = [s // HOP for s in samples]
    g = torch.Generator().manual_seed(SEED)
    codes = [[torch.randint(0, 1024, (1, rows, f), generator=g).cuda() for rows in (1, 2, 3)] for f in frames]
    timbre = [(0.3 * torch.randn(1, 1024, generator=g)).cuda() for _ in frames]
    waves = [synth.synth_waves(1, n, seed=SEED + j).cuda() for j, n in enumerate(samples)]
    audio_s = sum(frames) * HOP / SR

    def batches(order):
        out = []
        for i in range(0, len(order), args.batch):
            idx = order[i:i + args.batch]
            T = max(frames[j] for j in idx)
            packed = [torch.cat([torch.nn.functional.pad(codes[j][r], (0, T - frames[j])) for j in idx]) for r in range(3)]
            Ts = max(samples[j] for j in idx)
            x = torch.cat([torch.nn.functional.pad(waves[j], (0, Ts - samples[j])) for j in idx])
            out.append((idx, packed, torch.cat([timbre[j] for j in idx]), [frames[j] for j in idx], x, [samples[j] for j in idx]))
        return out

    arrival = batches(list(range(len(frames))))
    ordered = batches(sorted(range(len(frames)), key=lambda j: frames[j]))
    pad_frac = {name: 1.0 - sum(frames) / sum(len(b[0]) * max(b[3]) for b in bs)
                for name, bs in (("arrival", arrival), ("sorted", ordered))}

    # each call: (B = 1 call of utterance j, batched call of a batch) -> list of output tensors [lanes, ..., time]
    calls = {
        "encode": (lambda j: codec.encode(waves[j])[0], lambda bt: codec.encode(bt[4], lengths=bt[5])[0]),
        "forward": (lambda j: [codec.forward(waves[j])[0]], lambda bt: [codec.forward(bt[4], lengths=bt[5])[0]]),
        "decode": (lambda j: [codec.decode(codes[j], timbre[j])], lambda bt: [codec.decode(bt[1], bt[2], frames=bt[3])]),
        "convert": (lambda j: [vc.convert(codes[j][:2], timbre[j], use_p_code=False, n_c=2)],
                    lambda bt: [vc.convert(bt[1][:2], bt[2], use_p_code=False, n_c=2, frames=bt[3])]),
    }

    def run(call, mode):
        one, batched = call
        if mode == "b1":
            outs = [one(j) for j in range(len(frames))]
        else:
            outs = [batched(bt) for bt in (arrival if mode == "arrival" else ordered)]
        torch.cuda.synchronize()
        return outs

    results = {}
    for name, call in calls.items():
        for mode in ("b1", "arrival", "sorted"):          # warm-up: every shape of the timed rounds
            run(call, mode)
        best = {m: float("inf") for m in ("b1", "arrival", "sorted")}
        for _ in range(args.rounds):
            for mode in ("b1", "arrival", "sorted"):
                t0 = time.perf_counter()
                run(call, mode)
                best[mode] = min(best[mode], time.perf_counter() - t0)
        ref = run(call, "b1")
        checked = 0
        for mode, bs in (("arrival", arrival), ("sorted", ordered)):
            outs = run(call, mode)
            lanes = [(k, i) for k, b in enumerate(bs) for i in range(len(b[0]))]
            for k, i in random.Random(SEED + 1).sample(lanes, min(args.check, len(lanes))):
                j = bs[k][0][i]
                for got, want in zip(outs[k], ref[j]):
                    n = want.shape[-1]
                    assert torch.equal(got[i:i + 1, ..., :n], want), f"{name} {mode}: utterance {j} differs from B = 1"
                checked += 1
        results[name] = {m: round(audio_s / best[m], 1) for m in best}
        results[name]["lanes_checked_bit_equal"] = checked
        print(f"{name}: " + ", ".join(f"{m} {audio_s / best[m]:.1f} audio-s/s ({best[m] * 1e3:.0f} ms)" for m in best))

    card = card_info(0)
    card["sm_mhz_after"] = sm_clock_mhz(0)
    print(f"card: {card}")
    print(f"corpus: {args.utts} utterances, {audio_s:.1f} s of audio; padding arrival {pad_frac['arrival']:.3f}, "
          f"sorted {pad_frac['sorted']:.3f}")
    print(json.dumps({"metric": "ragged offline encode / forward / decode / convert, audio-s/s", "card": card, "utts": args.utts,
                      "batch": args.batch, "audio_s": round(audio_s, 1), "padding": {k: round(v, 4) for k, v in pad_frac.items()},
                      "results": results}))


if __name__ == "__main__":
    main()
