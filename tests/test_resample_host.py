"""Host-side checks of the sinc resampler: the float32 filter table against torchaudio's, the output and stream counts
against their formulas, unsupported rate pairs, and the fp64 restatement against torchaudio on the CPU."""
import math

import pytest
import torch

import facodec_b200 as fb
from facodec_b200 import _lib
from facodec_b200.modules import _rs_geometry
from oracle.resample import resample64

RATES = [8000, 11025, 16000, 22050, 32000, 44100, 48000, 96000, 192000]
PAIRS = [(r, 24000) for r in RATES] + [(24000, r) for r in RATES]


def _geometry(orig, new):
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    base = min(o, n) * 0.99
    width = math.ceil(6 * o / base)
    return o, n, width, 2 * width + o


@pytest.mark.parametrize("orig,new", PAIRS)
def test_table_equals_torchaudio(orig, new):
    F = pytest.importorskip("torchaudio.functional.functional")
    if orig == new:
        assert torch.equal(fb.resample_table(orig, new), torch.ones(1, 1))
        return
    ref, width = F._get_sinc_resample_kernel(orig, new, math.gcd(orig, new), dtype=torch.float32)
    tab = fb.resample_table(orig, new)
    assert torch.equal(tab, ref.squeeze(1))
    o, n, w, K = _rs_geometry(orig, new)
    assert (o, n, w, K) == _geometry(orig, new) and w == width and tab.shape == (n, K)
    assert K * n <= 65536


def test_largest_table():
    o, n, w, K = _rs_geometry(11025, 24000)
    assert K * n == 51520


@pytest.mark.parametrize("orig,new", [(44100, 24000), (24000, 48000), (16000, 24000), (24000, 11025), (24000, 24000)])
def test_out_len(orig, new):
    o, n, _, _ = _geometry(orig, new) if orig != new else (1, 1, 0, 1)
    L = _lib.load()
    for T in (0, 1, 2, 7, 299, 300, 11025, 96001):
        assert L.fac_resample_out_len(orig, new, T) == (n * T + o - 1) // o == fb.resample_length(orig, new, T)


@pytest.mark.parametrize("orig,new", [(44100, 24000), (24000, 48000), (48000, 24000), (24000, 11025), (8000, 24000)])
@pytest.mark.parametrize("quantum", [1, 300])
def test_stream_counts(orig, new, quantum):
    """A push returns the outputs whose whole window lies in the input so far, rounded down to the quantum; the stream's
    total is the offline length and the history a slot keeps stays within K + orig ceil((q - 1) / new)."""
    L = _lib.load()
    o, n, width, K = _geometry(orig, new)
    g = torch.Generator().manual_seed(orig + new + quantum)
    seen = emitted = full = 0
    for _ in range(200):
        seen += int(torch.randint(0, 900, (1,), generator=g))
        while full * o - width + K <= seen:          # block `full` has its whole window in the input
            full += 1
        avail = full * n                             # outputs of complete blocks: window [i o - width, i o - width + K)
        want = (avail - emitted) // quantum * quantum if avail > emitted else 0
        got = L.fac_resample_ready(orig, new, quantum, seen, emitted)
        assert got == want
        emitted += got
        assert emitted <= (n * seen + o - 1) // o
        hs = max(0, (emitted // n) * o - width)
        assert seen - hs <= K + o * ((quantum - 1 + n - 1) // n)
    final = L.fac_resample_out_len(orig, new, seen) - emitted
    assert final >= 0 and emitted + final == (n * seen + o - 1) // o


@pytest.mark.parametrize("orig,new", [(7999, 24000), (24000, 192001), (0, 24000), (24000, -1), (24001, 24000),
                                      (191999, 8000)])
def test_unsupported_rates(orig, new):
    assert _lib.load().fac_resample_geometry(orig, new, None) == -1
    assert _lib.load().fac_resample_out_len(orig, new, 100) < 0
    with pytest.raises(ValueError):
        fb.resample_table(orig, new)


@pytest.mark.parametrize("orig,new", [(44100, 24000), (24000, 48000), (24000, 11025)])
def test_oracle_matches_torchaudio_cpu(orig, new):
    """The fp64 restatement is torchaudio's sum: float32 torchaudio on the CPU lies within 2 (K + 1) 2^-24 of it per
    sample, relative to the sum of |terms|."""
    F = pytest.importorskip("torchaudio.functional")
    o, n, width, K = _rs_geometry(orig, new)
    x = torch.randn(2, 3001, generator=torch.Generator().manual_seed(5))
    y64, mass = resample64(x, o, n, width, fb.resample_table(orig, new))
    ta = F.resample(x, orig, new).double()
    assert ta.shape == y64.shape
    assert bool(((ta - y64).abs() <= 2 * (K + 1) * 2.0 ** -24 * mass + 1e-30).all())
