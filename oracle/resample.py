"""fp64 restatement of the sinc resampler (facodec_b200.resample, torchaudio.functional.resample's sum): for the float32
table h [new, K] of the reduced pair, y[j] = sum_k h[p][k] x[i orig - width + k] with i = j // new, p = j % new and x zero
outside [0, n), evaluated in float64.  Test-only."""
import torch


def resample64(x, orig, new, width, table):
    """x [B, T] (any float dtype) -> (y64 [B, ceil(new T / orig)], mass [B, same]: sum_k |h[p][k] x[.]|, for error bounds).
    orig / new / width are the reduced geometry (facodec_b200.modules._rs_geometry)."""
    x = x.detach().to("cpu", torch.float64)
    h = table.detach().to("cpu", torch.float64)
    B, T = x.shape
    K = h.shape[1]
    xp = torch.nn.functional.pad(x, (width, width + orig))
    win = xp.unfold(1, K, orig)                                   # [B, blocks, K]
    y = torch.einsum("bik,pk->bip", win, h).reshape(B, -1)
    mass = torch.einsum("bik,pk->bip", win.abs(), h.abs()).reshape(B, -1)
    n = (new * T + orig - 1) // orig
    return y[:, :n], mass[:, :n]
