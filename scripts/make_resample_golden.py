"""Writes tests/golden/resample_tables.npz: for every rate pair between 24 kHz and 8 / 11.025 / 16 / 22.05 / 32 / 44.1 / 48 /
96 / 192 kHz, three rows (phases 0, new // 2, new - 1) of torchaudio's float32 sinc_interp_hann table
(_get_sinc_resample_kernel(orig, new, gcd, dtype=torch.float32)), its width and the SHA-256 of the whole table's bytes, so
that facodec_b200.resample_table is checked against torchaudio where torchaudio is not installed.

    python scripts/make_resample_golden.py          # needs torchaudio
"""
import hashlib
import math
import os

import numpy as np
import torch
from torchaudio.functional.functional import _get_sinc_resample_kernel

RATES = [8000, 11025, 16000, 22050, 32000, 44100, 48000, 96000, 192000]
PAIRS = [(r, 24000) for r in RATES if r != 24000] + [(24000, r) for r in RATES if r != 24000]
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "resample_tables.npz")


def main():
    data = {}
    for o, n in PAIRS:
        tab, width = _get_sinc_resample_kernel(o, n, math.gcd(o, n), dtype=torch.float32)
        tab = tab.squeeze(1).contiguous().numpy()
        rows = sorted({0, tab.shape[0] // 2, tab.shape[0] - 1})
        key = "%d_%d" % (o, n)
        data[key + "_rows"] = np.array(rows, dtype=np.int64)
        data[key + "_taps"] = tab[rows]
        data[key + "_width"] = np.array(width, dtype=np.int64)
        data[key + "_sha256"] = np.array(hashlib.sha256(tab.tobytes()).hexdigest())
    np.savez_compressed(OUT, **data)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
