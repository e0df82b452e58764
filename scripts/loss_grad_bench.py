"""Forward + backward of train.py's mel criterion (train.py:155-163: MelSpectrogramLoss over windows 32 ... 2048, n_mels
5 ... 320, pow = 1, mag_weight = 0), gradient into the prediction only, as the generator step asks for it:

* facodec_b200.losses.MelSpectrogramLoss (fac_spectral_loss_grad: DFT GEMM, gradient kernel, transposed DFT GEMM and
  overlap-add per scale, all in the forward call; backward scales the saved gradient);
* the oracle restatement oracle.facodec_oracle.mel_spectrogram_loss in fp32 under torch autograd on the same GPU
  (torch.stft -> cuFFT), the library baseline.

Shapes: 8 x 24 000 samples (train.py's 80-frame segments, 8 per GPU) and 32 x 96 000 (the bench.py batch).  Per shape
the two paths alternate over --rounds rounds of --iters forward + backward steps each, timed with CUDA events after a
warm-up; the fastest round's per-step time is reported, with the DFT GEMM work computed from the shapes.

    python scripts/loss_grad_bench.py [--rounds 3] [--iters 10]

Prints the card, its power limit, its max SM clock and the SM clock sampled right after the timed rounds, then one JSON line.
Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from conv_layer_profile import card_info  # noqa: E402

SR = 24000
WINDOWS = [32, 64, 128, 256, 512, 1024, 2048]
N_MELS = [5, 10, 20, 40, 80, 160, 320]
SHAPES = [(8, 24000), (32, 96000)]


def sm_clock_mhz(index):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        return float(out.strip())
    except Exception as exc:     # the timings stand without it; say why it is missing
        return f"nvidia-smi: {exc}"


def dft_gflop(B, T, signals):
    """2 * MACs of the per-scale DFT GEMMs as executed, [rows][w] x [w][ld] (ld = 2 * (w / 2 + 1) rounded up to 128), over
    `signals` signals (frames T / hop + 1 each); the gradient GEMM [rows][ld] x [ld][w] does the same work."""
    f = 0.0
    for w in WINDOWS:
        frames = T // (w // 4) + 1
        ld = (2 * (w // 2 + 1) + 127) // 128 * 128
        f += 2.0 * signals * B * frames * w * ld
    return f / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds per shape")
    ap.add_argument("--iters", type=int, default=10, help="forward + backward steps per round")
    args = ap.parse_args()
    if args.rounds < 1 or args.iters < 1:
        ap.error("--rounds and --iters must be >= 1")

    import torch
    from facodec_b200 import losses, synth
    from oracle import facodec_oracle as O

    assert torch.cuda.is_available(), "loss_grad_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    ours = losses.MelSpectrogramLoss(n_mels=N_MELS, window_lengths=WINDOWS, mel_fmin=[0.0] * 7, mel_fmax=[None] * 7, pow=1.0,
                                     mag_weight=0.0, clamp_eps=1e-5)

    def oracle(p, y):
        return O.mel_spectrogram_loss(p, y, SR, n_mels=N_MELS, window_lengths=WINDOWS, mel_fmin=[0.0] * 7, mel_fmax=[None] * 7,
                                      pow=1.0, mag_weight=0.0)

    res = {"criterion": "train.py:155-163 MelSpectrogramLoss, gradient into the prediction", "rounds": args.rounds,
           "iters": args.iters, "shapes": []}
    for B, T in SHAPES:
        x, y = synth.synth_loss_pair(B, T, seed=9)
        pred = x.cuda().requires_grad_(True)
        ref = y.cuda()

        def step(fn):
            pred.grad = None
            fn(pred, ref).backward()

        def timed(fn):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                step(fn)
            b.record()
            b.synchronize()
            return a.elapsed_time(b) / args.iters

        for _ in range(2):
            step(ours)
            step(oracle)
        torch.cuda.synchronize()
        ms = {"ours": [], "torch_cufft": []}
        for _ in range(args.rounds):
            ms["ours"].append(timed(ours))
            ms["torch_cufft"].append(timed(oracle))
        clock = sm_clock_mhz(0)
        # the two gradients on this shape, for the record (normwise relative difference, fp32 both)
        pred.grad = None
        ours(pred, ref).backward()
        g1 = pred.grad.clone()
        pred.grad = None
        oracle(pred, ref).backward()
        g2 = pred.grad.clone()
        rel = float((g1 - g2.reshape(g1.shape)).norm() / g2.norm())
        row = {"B": B, "T": T, "dft_gemm_gflop": {"forward_both_signals": round(dft_gflop(B, T, 2), 1),
                                                  "gradient_dx_only": round(dft_gflop(B, T, 1), 1)},
               "sm_clock_mhz_after_rounds": clock, "grad_rel_diff_vs_torch": f"{rel:.2e}"}
        for k, v in ms.items():
            row[k] = {"ms_per_step": [round(t, 3) for t in v], "fastest": round(min(v), 3)}
        res["shapes"].append(row)

    card = card_info(0)
    res["card"] = card
    print(f"card: {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['max_sm_mhz']} MHz"
          + (f" ({card['error']})" if "error" in card else ""))
    for r in res["shapes"]:
        print(f"B={r['B']} T={r['T']}: ours {r['ours']['fastest']} ms/step, torch/cuFFT {r['torch_cufft']['fastest']} ms/step "
              f"(SM clock after the rounds {r['sm_clock_mhz_after_rounds']} MHz)")
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
