"""Per-layer device time of the codec forward at the bench.py workload (32 x 4 s utterances, seeded synthetic inputs and
weights), from the library's own launch profiler: CUDA events around every launch, summed per call site over the
profiled steps.  bench.py reports only kernel-family totals; this shows which layers the time goes to.

    python scripts/conv_layer_profile.py [--steps 2] [--warmup 2] [--top 0]

Prints the card, its power limit and max SM clock, then one row per call site sorted by time: ms per step, algorithmic
GFLOP per step (2 x MACs) and TFLOP/s.  Events around every launch add a little host overhead; take step times from
bench.py, not from this script.  Needs a CUDA device.
"""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BATCH = 32                  # bench.py BATCH_PER_GPU
UTT_SAMPLES = 24000 * 4     # bench.py UTT_SAMPLES
SEED = 114514               # bench.py input seed of rank 0


def card_info(index):
    import torch
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "max_sm_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        pl, mx = [f.strip() for f in out.strip().split(",")[:2]]
        info["power_limit_w"], info["max_sm_mhz"] = float(pl), float(mx)
    except Exception as exc:     # the timings stand without it; say why it is missing
        info["error"] = f"nvidia-smi: {exc}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2, help="profiled forward passes (the table is per step)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--top", type=int, default=0, help="print only the N slowest call sites (0 = all)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")

    import torch
    import facodec_b200 as fb
    from facodec_b200 import synth

    assert torch.cuda.is_available(), "conv_layer_profile.py needs a CUDA device"
    torch.cuda.set_device(0)
    sds = synth.synth_state_dicts(0)
    model = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        model[k].load_state_dict(sds[k])
        model[k].eval()
    codec = fb.Codec(model)
    x = synth.synth_waves(BATCH, UTT_SAMPLES, seed=SEED).contiguous().cuda()

    for _ in range(args.warmup):
        codec.forward(x, n_c=2)
    torch.cuda.synchronize()
    L, h = codec.engine.L, codec.engine.handle
    L.fac_profile_reset(h)
    L.fac_profile_enable(h, 1)
    for _ in range(args.steps):
        codec.forward(x, n_c=2)
    torch.cuda.synchronize()
    L.fac_profile_enable(h, 0)
    n = L.fac_profile_dump(h, None, 0)
    buf = ctypes.create_string_buffer(n)
    L.fac_profile_dump(h, buf, n)
    L.fac_profile_reset(h)

    rows = []
    for line in buf.value.decode().splitlines():
        key, ms, gflop, _gbytes, launches = line.split("\t")
        family, _, site = key.partition(":")
        rows.append((family, site or "-", float(ms) / args.steps, float(gflop) / args.steps, int(launches) // args.steps))
    rows.sort(key=lambda r: -r[2])
    total = sum(r[2] for r in rows)

    card = card_info(0)
    print(f"card: {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['max_sm_mhz']} MHz"
          + (f" ({card['error']})" if "error" in card else ""))
    print(f"workload: {BATCH} x 4 s utterances, n_c = 2; {args.steps} profiled steps after {args.warmup} warm-up; "
          f"profiled launches sum to {total:.2f} ms per step")
    fams = {}
    for fam, _, ms, gf, nl in rows:
        a = fams.setdefault(fam, [0.0, 0.0, 0])
        a[0] += ms; a[1] += gf; a[2] += nl
    print(f"{'family':<12} {'ms/step':>9} {'share':>6} {'GFLOP':>9} {'TFLOP/s':>8} {'launches':>8}")
    for fam, (ms, gf, nl) in sorted(fams.items(), key=lambda kv: -kv[1][0]):
        print(f"{fam:<12} {ms:9.3f} {ms / total:6.1%} {gf:9.1f} {gf / ms if ms > 0 else 0.0:8.1f} {nl:8d}")
    print()
    print(f"{'family':<10} {'call site':<52} {'ms/step':>9} {'share':>6} {'GFLOP':>9} {'TFLOP/s':>8} {'launches':>8}")
    for fam, site, ms, gf, nl in rows[:args.top or None]:
        print(f"{fam:<10} {site:<52} {ms:9.3f} {ms / total:6.1%} {gf:9.1f} {gf / ms if ms > 0 else 0.0:8.1f} {nl:8d}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
