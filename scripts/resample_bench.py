"""Sample-rate conversion on the GPU (facodec_b200.resample, ResamplePool, and sessions at 48 kHz in the stream pools):

* offline: resample() of --batch x --seconds of audio for every pair between 24 kHz and 8 / 11.025 / 16 / 22.05 / 32 / 44.1 /
  48 / 96 / 192 kHz, against torchaudio.transforms.Resample(dtype=torch.float32) (the same float32 table, built once) on the
  same GPU with cuDNN TF32 off.  CUDA events, the fastest of --rounds alternating rounds; the max |difference| between
  the two outputs, which comes from the order of the sums alone (cuDNN's conv1d against one fixed fmaf chain per output).
* pool: one ResamplePool.push step of S sessions of mixed pairs fed 0.25 s chunks, S in --sessions; wall time per step
  (host clock around a device synchronise), median over --steps steps.
* serving: --callers live callers through CodecStreamPool.encode_codes + VoiceConversionPool.convert per 0.25 s step, once
  with 48 kHz callers (both pools resample) and once with the same audio at 24 kHz, alternating; median step time of each
  and the resampling share 1 - t24 / t48.

    python scripts/resample_bench.py [--batch 32] [--seconds 4] [--rounds 5] [--sessions 32,128] [--callers 32]
    python scripts/resample_bench.py --rehearse      # no GPU: argument parsing and the fp64 oracle path at a tiny size

Prints the card, its power limit and max SM clock, then one JSON line (also written to --out when given).  Synthetic
checkpoints (seed 0) for the serving part.
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

RATES = [8000, 11025, 16000, 22050, 32000, 44100, 48000, 96000, 192000]
PAIRS = [(r, 24000) for r in RATES if r != 24000] + [(24000, r) for r in RATES if r != 24000]
POOL_PAIRS = [(48000, 24000), (44100, 24000), (16000, 24000), (24000, 48000), (24000, 16000), (8000, 24000)]


def rehearse(args):
    """The oracle path on the CPU at a tiny size: the tables against the stored torchaudio digests, the fp64 restatement's
    output mass, and (where torchaudio is installed) the restatement against torchaudio's float32 resample."""
    import hashlib
    import numpy as np
    import facodec_b200 as fb
    from facodec_b200.modules import _rs_geometry
    from oracle.resample import resample64
    try:
        import torchaudio.functional as F
    except ImportError:
        F = None
    golden = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                                  "resample_tables.npz"))
    out = {}
    x = torch.randn(2, 2000, generator=torch.Generator().manual_seed(0))
    for o, n in PAIRS[:3] + PAIRS[-3:]:
        ro, rn, width, K = _rs_geometry(o, n)
        tab = fb.resample_table(o, n)
        y64, mass = resample64(x, ro, rn, width, tab)
        r = {"table_matches_golden": hashlib.sha256(tab.numpy().tobytes()).hexdigest() == str(golden["%d_%d_sha256" % (o, n)]),
             "fp32_bound": float(((K + 1) * 2.0 ** -24 * mass).max())}
        if F is not None:
            r["torchaudio_max_abs_diff"] = float((F.resample(x, o, n).double() - y64).abs().max())
        out["%d->%d" % (o, n)] = r
    print(json.dumps({"rehearsal": "cpu oracle path", "pairs": out}))


def events_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def bench_offline(args, fb):
    import torchaudio
    res = {}
    torch.backends.cudnn.allow_tf32 = False          # torchaudio's conv1d would otherwise run its taps in TF32
    for o, n in PAIRS:
        if o == n:
            continue
        x = torch.randn(args.batch, int(o * args.seconds), generator=torch.Generator().manual_seed(o + n)).cuda()
        ta = torchaudio.transforms.Resample(o, n, dtype=torch.float32).cuda()     # F.resample's float32 table
        ours = lambda: fb.resample(x, o, n)
        theirs = lambda: ta(x)
        ours(); theirs()
        torch.cuda.synchronize()
        t_ours, t_ta = [], []
        for _ in range(args.rounds):
            t_ours.append(events_ms(ours, 5))
            t_ta.append(events_ms(theirs, 5))
        diff = float((ours() - theirs()).abs().max())
        res["%d->%d" % (o, n)] = {"ms": min(t_ours), "torchaudio_ms": min(t_ta), "max_abs_diff": diff}
    return res


def bench_pool(args, fb):
    res = {}
    for S in [int(s) for s in args.sessions.split(",")]:
        pool = fb.ResamplePool(S)
        ss = [pool.open(*POOL_PAIRS[i % len(POOL_PAIRS)]) for i in range(S)]
        g = torch.Generator().manual_seed(S)
        chunks = {s: torch.randn(1, POOL_PAIRS[i % len(POOL_PAIRS)][0] // 4, generator=g).cuda() for i, s in enumerate(ss)}
        times = []
        for k in range(args.steps + 2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pool.push(chunks)
            torch.cuda.synchronize()
            if k >= 2:
                times.append((time.perf_counter() - t0) * 1e3)
        pool.close()
        res[str(S)] = {"median_step_ms": statistics.median(times)}
    return res


def bench_serving(args, fb):
    from facodec_b200 import synth
    codec = fb.build_model()
    sds = synth.synth_state_dicts(0)
    for k in ("encoder", "quantizer", "decoder"):
        codec[k].load_state_dict(sds[k])
        codec[k].eval()
    red = fb.build_model(stage="redecoder")
    rsd = synth.synth_redecoder_state_dicts(0)
    for k in ("encoder", "decoder"):
        red[k].load_state_dict(rsd[k])
        red[k].eval()
    S, steps = args.callers, args.serving_steps
    timbre = torch.randn(1, 1024, generator=torch.Generator().manual_seed(1)).cuda()
    w24 = synth.synth_waves(S, 6000 * steps, seed=3).cuda()
    w48 = fb.resample(w24, 24000, 48000)

    def run(rate, wave, chunk):
        tx = fb.CodecStreamPool(codec, capacity=S)
        vc = fb.VoiceConversionPool(red, capacity=S)
        ts = [tx.open(sample_rate=rate) for _ in range(S)]
        vs = [vc.open(timbre, sample_rate=rate) for _ in range(S)]
        times = []
        for k in range(steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            codes = tx.encode_codes({s: wave[i:i + 1, :, k * chunk:(k + 1) * chunk] for i, s in enumerate(ts)})
            feed = {vs[i]: codes[s] for i, s in enumerate(ts) if codes[s][0].shape[2] > 0}
            if feed:
                vc.convert(feed)
            torch.cuda.synchronize()
            if k >= 2:
                times.append((time.perf_counter() - t0) * 1e3)
        tx.close()
        vc.close()
        return statistics.median(times)

    t24, t48 = [], []
    for _ in range(args.rounds):
        t24.append(run(24000, w24, 6000))
        t48.append(run(48000, w48, 12000))
    m24, m48 = min(t24), min(t48)
    return {"callers": S, "step_ms_24k": m24, "step_ms_48k": m48, "resample_share": 1 - m24 / m48}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=4.0)
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds; the fastest (offline) / best median counts")
    ap.add_argument("--sessions", default="32,128", help="comma-separated ResamplePool sizes")
    ap.add_argument("--steps", type=int, default=40, help="timed ResamplePool steps")
    ap.add_argument("--callers", type=int, default=32, help="serving callers (0: skip the serving part)")
    ap.add_argument("--serving-steps", type=int, default=16, help="0.25 s steps per serving run")
    ap.add_argument("--rehearse", action="store_true", help="no GPU: the CPU oracle path at a tiny size")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.rounds < 1 or args.batch < 1 or args.seconds <= 0 or args.steps < 1 or args.serving_steps < 3:
        ap.error("rounds, batch, steps >= 1, seconds > 0, serving-steps >= 3")
    if args.rehearse:
        return rehearse(args)
    if not torch.cuda.is_available():
        sys.exit("resample_bench.py needs a CUDA device (--rehearse runs the CPU part)")
    import facodec_b200 as fb
    from conv_layer_profile import card_info
    card = card_info(0)
    print("card:", card)
    out = {"card": card, "offline": bench_offline(args, fb), "pool": bench_pool(args, fb)}
    if args.callers > 0:
        out["serving"] = bench_serving(args, fb)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
