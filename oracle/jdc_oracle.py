"""fp64 CPU restatement of JDCNet's eval-mode forward (modules/JDC/model.py:102-137 with num_class = 1) and of train.py's
F0 and energy targets (train.py:214-254, modules/commons.py:176-181).

`jdc_forward(sd, x, lengths=None, dtype=torch.float64)` takes the reference state dict and mel x [B, 1, 80, T] and returns
(F0 [B, T], GAN_feature [B, 256, 10, T], poolblock_out [B, 256, T, 2], taps).  BatchNorm uses its running statistics
and Dropout is the identity.  With `lengths`, lane b is computed on its own first lengths[b] frames (as a B = 1 call) and
its outputs past them are zero.  `dtype=torch.float32` gives the same computation in fp32, the yardstick of the tests'
error bars.  `taps` holds every block's output in the reference's NCHW layout ([B, C, T, F]).
"""
import torch
import torch.nn.functional as F

_BLOCKS = (("res_block1", 64, 128), ("res_block2", 128, 192), ("res_block3", 192, 256))


def _bn(sd, prefix, x):
    g = sd[prefix + ".weight"].to(x.dtype)
    b = sd[prefix + ".bias"].to(x.dtype)
    m = sd[prefix + ".running_mean"].to(x.dtype)
    v = sd[prefix + ".running_var"].to(x.dtype)
    return F.batch_norm(x, m, v, g, b, training=False, eps=1e-5)


def _lrelu(x):
    return F.leaky_relu(x, 0.01)


def _conv(sd, key, x, pad):
    return F.conv2d(x, sd[key].to(x.dtype), padding=pad)


def lstm_dir(wih, whh, bih, bhh, x, reverse=False):
    """One direction of nn.LSTM (gate order i, f, g, o) over x [T, 512] -> [T, H]."""
    H = whh.shape[1]
    h = torch.zeros(H, dtype=x.dtype)
    c = torch.zeros(H, dtype=x.dtype)
    xg = x @ wih.t() + bih + bhh
    out = torch.zeros(x.shape[0], H, dtype=x.dtype)
    steps = range(x.shape[0] - 1, -1, -1) if reverse else range(x.shape[0])
    for t in steps:
        g = xg[t] + whh @ h
        i, f, gg, o = torch.sigmoid(g[:H]), torch.sigmoid(g[H:2 * H]), torch.tanh(g[2 * H:3 * H]), torch.sigmoid(g[3 * H:])
        c = f * c + i * gg
        h = o * torch.tanh(c)
        out[t] = h
    return out


def _forward_one(sd, x, dtype):
    """x [1, 1, 80, T] -> the eval-mode outputs and the block taps of one utterance."""
    taps = {}
    x = x.to(dtype).transpose(-1, -2)                                     # [1, 1, T, 80]
    h = _lrelu(_bn(sd, "conv_block.1", _conv(sd, "conv_block.0.weight", x, 1)))
    taps["conv_in"] = h
    h = _conv(sd, "conv_block.3.weight", h, 1)
    taps["conv_block"] = h
    for name, _, _ in _BLOCKS:
        xp = F.max_pool2d(_lrelu(_bn(sd, name + ".pre_conv.0", h)), (1, 2))
        taps[name + ".pre"] = xp
        a = _lrelu(_bn(sd, name + ".conv.1", _conv(sd, name + ".conv.0.weight", xp, 1)))
        taps[name + ".conv1"] = a
        h = _conv(sd, name + ".conv.3.weight", a, 1) + _conv(sd, name + ".conv1by1.weight", xp, 0)
        taps[name] = h
    p = _lrelu(_bn(sd, "pool_block.0", h))                               # [1, 256, T, 10]
    gan = p.transpose(-1, -2)
    pool = F.max_pool2d(p, (1, 4))                                        # [1, 256, T, 2]
    T = x.shape[2]
    seq = pool.permute(0, 2, 1, 3).reshape(T, 512)
    taps["lstm_in"] = seq
    d = {}
    for sfx, rev in (("_l0", False), ("_l0_reverse", True)):
        w = [sd["bilstm_classifier." + n + sfx].to(dtype) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        d[rev] = lstm_dir(*w, seq, reverse=rev)
    taps["lstm.fwd"], taps["lstm.rev"] = d[False], d[True]
    y = torch.cat([d[False], d[True]], dim=1) @ sd["classifier.weight"].to(dtype).t() + sd["classifier.bias"].to(dtype)
    return y.abs().reshape(1, T), gan, pool, taps


def jdc_forward(sd, x, lengths=None, dtype=torch.float64):
    B, T = x.shape[0], x.shape[-1]
    lens = [T] * B if lengths is None else [int(v) for v in lengths]
    f0 = torch.zeros(B, T, dtype=dtype)
    gan = torch.zeros(B, 256, 10, T, dtype=dtype)
    pool = torch.zeros(B, 256, T, 2, dtype=dtype)
    taps = []
    for b in range(B):
        L = lens[b]
        fb, gb, pb, tb = _forward_one(sd, x[b:b + 1, :, :, :L], dtype)
        f0[b, :L], gan[b, :, :, :L], pool[b, :, :L] = fb[0], gb[0], pb[0]
        taps.append(tb)
    return f0, gan, pool, taps


def f0_targets(f0, lengths=None):
    """train.py:223-251 (norm_f0) per lane in fp64 -> (targets [B, T], glob_f0 [B]); frames past lengths[b] are -10."""
    f0 = f0.to(torch.float64)
    B, T = f0.shape
    out = torch.full((B, T), -10.0, dtype=torch.float64)
    glob = torch.zeros(B, dtype=torch.float64)
    for b in range(B):
        L = T if lengths is None else int(lengths[b])
        row = f0[b, :L]
        voiced = row > 5.0
        if int(voiced.sum()) == 0:
            continue
        lf = row[voiced].log2()
        mean, std = lf.mean(), lf.std()
        seq = torch.full((L,), -10.0, dtype=torch.float64)
        seq[voiced] = (lf - mean) / std
        seq[torch.isnan(seq) | torch.isinf(seq)] = -10.0
        out[b, :L] = seq
        glob[b] = mean
    return out, glob


def log_norm(mel):
    """modules/commons.py:176-181 with mean -4, std 4 over the bins of mel [B, 80, T] -> [B, T], in fp64."""
    m = mel.to(torch.float64)
    return torch.log(torch.exp(m * 4 - 4).norm(dim=1))
