"""Voice-conversion pool steps with mixed conversion modes and mid-call voice switches: synthetic checkpoint 0, 20-frame
(0.25 s) chunks of random codes, every caller a --seconds utterance starting at step i % 8 (the staggered joins and leaves
of stream_pool_bench.py).  Three cases, alternating in one process (--rounds rounds each):

* uniform: every session in the pool's mode (use_p_code False, n_c 1);
* mixed: sessions cycle through (use_p_code, n_c) in {(0,1), (1,1), (0,2), (1,2)}, sharing launches;
* switch: as uniform, and before the middle step a quarter of the callers (i % 4 == 0) switch voice (set_timbre); the
  switched sessions' step recomputes their latent history on a wider window.

Wall time per step, host clock around a device synchronise: median and p99 over all steps, and the switch step (with its
set_timbre calls) against the same step of the uniform case.  Each case's outputs are checked against the offline
VoiceConverter.convert (the switch case against the splice of two conversions).  S in --callers (default 32, 128).

    python scripts/vc_switch_bench.py [--rounds 3] [--seconds 4] [--callers 32,128]

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

from conv_layer_profile import card_info  # noqa: E402
from stream_vc_bench import pct, sm_clock_mhz  # noqa: E402

SR, HOP, CHUNK = 24000, 300, 20
LOOKAHEAD = 44
MODES = [(False, 1), (True, 1), (False, 2), (True, 2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="rounds of each case, alternating")
    ap.add_argument("--seconds", type=float, default=4.0, help="length of every caller's utterance")
    ap.add_argument("--callers", default="32,128", help="comma-separated S")
    args = ap.parse_args()
    callers = [int(s) for s in args.callers.split(",")]
    if args.rounds < 1 or args.seconds * SR < 4 * CHUNK * HOP or min(callers) < 4:
        ap.error("--rounds >= 1, --seconds >= 1, callers >= 4")

    import torch
    import facodec_b200 as fb
    from facodec_b200 import synth

    assert torch.cuda.is_available(), "vc_switch_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    rsds = synth.synth_redecoder_state_dicts(0)
    vc_model = fb.build_model(stage="redecoder")
    for k in ("encoder", "decoder"):
        vc_model[k].load_state_dict(rsds[k])
        vc_model[k].eval()

    nchunks = int(args.seconds * SR) // (CHUNK * HOP)
    T = nchunks * CHUNK
    smax = max(callers)
    g = torch.Generator().manual_seed(1234)
    cps = torch.randint(0, 1024, (smax, 1, T), generator=g).cuda()
    ccs = torch.randint(0, 1024, (smax, 2, T), generator=g).cuda()
    timbres = torch.randn(smax, 1024, generator=g).cuda()
    others = torch.randn(smax, 1024, generator=g).cuda()

    def sync_ms(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    def schedule(S):
        return [[(i, step - i % 8) for i in range(S) if 0 <= step - i % 8 < nchunks] for step in range(nchunks + 7)]

    mid = (nchunks + 7) // 2

    def run(S, case):
        """-> (outputs, step times, time of step `mid`)."""
        ys, times = [[] for _ in range(S)], []
        with fb.VoiceConversionPool(vc_model, capacity=S, use_p_code=False, n_c=1) as vc:
            vs = {}

            def step(k_step, feed):
                for i, k in feed:
                    if k == 0:
                        mode = dict(zip(("use_p_code", "n_c"), MODES[i % 4])) if case == "mixed" else {}
                        vs[i] = vc.open(timbres[i:i + 1], **mode)
                if case == "switch" and k_step == mid:
                    for i, k in feed:
                        if i % 4 == 0 and k > 0:
                            vc.set_timbre(vs[i], others[i:i + 1])
                out = vc.convert({vs[i]: [cps[i:i + 1, :, k * CHUNK:(k + 1) * CHUNK], ccs[i:i + 1, :, k * CHUNK:(k + 1) * CHUNK]]
                                  for i, k in feed})
                for i, _ in feed:
                    ys[i].append(out[vs[i]])
                ending = [i for i, k in feed if k == nchunks - 1]
                if ending:
                    tail = vc.finish([vs[i] for i in ending])
                    for i in ending:
                        ys[i].append(tail[vs[i]])
                        vc.close(vs[i])

            for k_step, feed in enumerate(schedule(S)):
                times.append(sync_ms(lambda: step(k_step, feed)))
        return [torch.cat(y, dim=2) for y in ys], times, times[mid]

    def check(S, case, ys):
        conv = fb.VoiceConverter(vc_model)
        for i in range(S):
            mode = dict(zip(("use_p_code", "n_c"), MODES[i % 4])) if case == "mixed" else dict(use_p_code=False, n_c=1)
            ref = conv.convert([cps[i:i + 1], ccs[i:i + 1]], timbres[i:i + 1], **mode)
            k = mid - i % 8
            if case == "switch" and i % 4 == 0 and 0 < k < nchunks:
                Yf = max(k * CHUNK - LOOKAHEAD, 0)
                new = conv.convert([cps[i:i + 1], ccs[i:i + 1]], others[i:i + 1], **mode)
                ref = torch.cat([ref[:, :, :HOP * Yf], new[:, :, HOP * Yf:]], dim=2)
            if not torch.equal(ys[i], ref):
                return False
        return True

    cases = ("uniform", "mixed", "switch")
    for case in cases:                                   # warm-up: sizes the workspaces, loads the modules
        run(min(callers), case)
    res = {"chunk_frames": CHUNK, "seconds_each": T * HOP / SR, "rounds": args.rounds, "callers": {}}
    for S in callers:
        ms = {c: [] for c in cases}
        mids = {c: [] for c in cases}
        equal = {c: True for c in cases}
        for r in range(args.rounds):
            for c in cases:
                ys, t, tm = run(S, c)
                ms[c] += t
                mids[c].append(tm)
                if r == 0:
                    equal[c] = check(S, c, ys)
        out = {}
        for c in cases:
            out[c] = {"step_ms_median": round(pct(ms[c], 0.5), 3), "step_ms_p99": round(pct(ms[c], 0.99), 3),
                      "mid_step_ms_median": round(pct(mids[c], 0.5), 3), "equal_offline": equal[c]}
        out["switched_sessions"] = sum(1 for i, k in schedule(S)[mid] if i % 4 == 0 and k > 0)
        res["callers"][S] = out
    clock = sm_clock_mhz(0)
    card = card_info(0)
    print(f"card: {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['max_sm_mhz']} MHz, "
          f"SM clock after the timed rounds {clock} MHz" + (f" ({card['error']})" if "error" in card else ""))
    res["card"], res["sm_clock_mhz_after_rounds"] = card, clock
    print(json.dumps(res))
    return 0 if all(v["equal_offline"] for r in res["callers"].values() for k, v in r.items() if isinstance(v, dict)) else 1


if __name__ == "__main__":
    sys.exit(main())
