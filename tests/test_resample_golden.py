"""facodec_b200.resample_table against stored rows and digests of torchaudio's float32 tables (tests/golden/
resample_tables.npz, written by scripts/make_resample_golden.py), so the table the GPU contracts and the fp64 oracle rely on
is checked with or without torchaudio installed."""
import hashlib

import numpy as np
import pytest

import facodec_b200 as fb
from facodec_b200.modules import _rs_geometry
from conftest import load_golden

RATES = [8000, 11025, 16000, 22050, 32000, 44100, 48000, 96000, 192000]
PAIRS = [(r, 24000) for r in RATES if r != 24000] + [(24000, r) for r in RATES if r != 24000]


@pytest.mark.parametrize("orig,new", PAIRS)
def test_table_equals_stored_torchaudio_table(orig, new):
    g = load_golden("resample_tables")
    key = "%d_%d" % (orig, new)
    tab = fb.resample_table(orig, new).numpy()
    assert _rs_geometry(orig, new)[2] == int(g[key + "_width"])
    assert np.array_equal(tab[g[key + "_rows"]], g[key + "_taps"])
    assert hashlib.sha256(np.ascontiguousarray(tab).tobytes()).hexdigest() == str(g[key + "_sha256"])
