"""Times JDCNet.forward + f0_targets (facodec_b200) against the fp32 torch restatement (oracle/jdc_oracle.py run on the
same GPU with cuDNN, TF32 off) at 32 x 4 s (320 frames each) and at train.py's shape (4 x 80 frames).

    python scripts/jdc_bench.py [--reps 20] [--out FILE]

Prints one JSON line per shape (and writes them to --out when given); times are the best of --reps calls, timed with
CUDA events.  FLOP count from the shapes, per frame:
  3x3 convs  2 * 9 * (80 * 64 * 64 + 40 * (64 * 128 + 128 * 128) + 20 * (128 * 192 + 192 * 192) + 10 * (192 * 256 + 256 * 256))
  1x1 convs  2 * (40 * 64 * 128 + 20 * 128 * 192 + 10 * 192 * 256)
  BiLSTM     2 * 2 * 4 * 256 * (512 + 256)
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import facodec_b200 as fb  # noqa: E402
from facodec_b200 import synth  # noqa: E402
from oracle import jdc_oracle as O  # noqa: E402

CONV3 = 2 * 9 * (80 * 64 * 64 + 40 * (64 * 128 + 128 * 128) + 20 * (128 * 192 + 192 * 192) + 10 * (192 * 256 + 256 * 256))
CONV1 = 2 * (40 * 64 * 128 + 20 * 128 * 192 + 10 * 192 * 256)
LSTM = 2 * 2 * 4 * 256 * (512 + 256)
FLOP_PER_FRAME = CONV3 + CONV1 + LSTM


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def _torch_fp32(sd, x):
    """The restatement's layers in fp32 on the GPU (batched; the LSTM through nn.LSTM)."""
    import torch.nn.functional as F
    d = {k: v.cuda().float() for k, v in sd.items()}
    lstm = torch.nn.LSTM(512, 256, batch_first=True, bidirectional=True).cuda()
    lstm.load_state_dict({k[len("bilstm_classifier."):]: v for k, v in d.items() if k.startswith("bilstm_classifier.")})

    def run():
        with torch.no_grad():
            h = x.transpose(-1, -2)
            h = O._lrelu(O._bn(d, "conv_block.1", O._conv(d, "conv_block.0.weight", h, 1)))
            h = O._conv(d, "conv_block.3.weight", h, 1)
            for name, _, _ in O._BLOCKS:
                xp = F.max_pool2d(O._lrelu(O._bn(d, name + ".pre_conv.0", h)), (1, 2))
                a = O._lrelu(O._bn(d, name + ".conv.1", O._conv(d, name + ".conv.0.weight", xp, 1)))
                h = O._conv(d, name + ".conv.3.weight", a, 1) + O._conv(d, name + ".conv1by1.weight", xp, 0)
            p = F.max_pool2d(O._lrelu(O._bn(d, "pool_block.0", h)), (1, 4))
            y, _ = lstm(p.permute(0, 2, 1, 3).reshape(x.shape[0], x.shape[-1], 512))
            return (y @ d["classifier.weight"].t() + d["classifier.bias"]).abs().squeeze(-1)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("jdc_bench.py needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = synth.synth_jdc(0)
    net = fb.JDCNet()
    net.load_state_dict(sd)
    net.eval()
    rows = []
    for B, T in ((32, 320), (4, 80)):
        x = (torch.randn(B, 1, 80, T, generator=torch.Generator().manual_seed(0)) * 0.6 - 0.5).cuda()

        def ours():
            f0, _, _ = net(x)
            fb.f0_targets(f0)
        ms = _time(ours, args.reps)
        ms_t = _time(_torch_fp32(sd, x), args.reps)
        flop = FLOP_PER_FRAME * B * T
        rows.append(dict(shape=f"{B}x{T}", frames=B * T, jdc_ms=round(ms, 3), torch_fp32_ms=round(ms_t, 3),
                         tflops=round(flop / ms / 1e9, 2), mflop_per_frame=round(FLOP_PER_FRAME / 1e6, 2)))
    # read in the same run as the timings: the card, its power limit and its maximum SM clock
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    for r in rows:
        r["card"] = card
        print(json.dumps(r))
    if args.out:
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in rows))


if __name__ == "__main__":
    main()
