"""Library baseline (SURVEY.md 8d): the reference's own ATen call sequence (the oracle restatement, i.e. what the
reference's nn.Modules execute) run by PyTorch eager on the same GPU in fp32 with TF32 disabled, at BASELINE
configs[1] (32 x 4 s), timed beside this repo's path.  Informational numbers are printed (pytest -s); the assertions
only pin that both paths agree (cuDNN picks its own summation orders, so a handful of near-tied VQ decisions may differ
between eager-GPU and the CPU reference -- this repo matches the CPU reference bit for bit, see test_gpu_parity.py).
The file name sorts last so that `pytest -x` reaches it after the parity tests."""
import pytest
import torch

from conftest import state_dicts

pytestmark = pytest.mark.gpu


def test_reference_ops_eager_on_gpu_baseline(built_lib):
    import facodec_b200 as fb
    from facodec_b200 import synth
    from oracle import facodec_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    sds = state_dicts(0)
    sds_gpu = {k: {n: t.to(dev) for n, t in sd.items()} for k, sd in sds.items()}
    x = synth.synth_waves(32, 96000).to(dev)

    def timed(fn, n):
        fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            out = fn()
        b.record()
        torch.cuda.synchronize()
        return out, a.elapsed_time(b) / n

    try:
        with torch.no_grad():
            (zo, qo, yo), ms_eager = timed(lambda: O.codec_forward(sds_gpu, x, n_c=2), 2)
    except RuntimeError as e:      # e.g. out of memory on a smaller device: the baseline is informational
        pytest.skip(f"eager baseline could not run here: {e}")
    m = fb.build_model()
    for k in ("encoder", "quantizer", "decoder"):
        m[k].load_state_dict(sds[k])
        m[k].eval()
    codec = fb.Codec(m)
    (y, codes, timbre), ms_ours = timed(lambda: codec.forward(x, n_c=2), 3)
    audio_s = 32 * 4.0
    total = sum(c.numel() for c in codes)
    diff = sum(int((a != b).sum()) for a, b in zip(codes, qo[5]))
    rms = float(((y.double() - yo.double()) ** 2).mean().sqrt())
    print(f"\nEAGER-GPU baseline (torch {torch.__version__}, fp32, TF32 off): {ms_eager:.1f} ms/step = {audio_s / ms_eager * 1e3:.0f} audio-s/s; "
          f"this repo: {ms_ours:.1f} ms/step = {audio_s / ms_ours * 1e3:.0f} audio-s/s ({ms_eager / ms_ours:.2f}x); "
          f"VQ indices differing between the two GPU paths: {diff} of {total}; waveform rms diff {rms:.2e}")
    assert diff <= total // 500          # near-ties only
    assert rms <= 2e-3 or diff > 0       # identical codes => waveforms agree to fp32 noise
