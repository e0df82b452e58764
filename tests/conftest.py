import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a; select with -m gpu)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def built_lib():
    """The in-tree C-ABI library, (re)built if stale (nvcc cross-compiles without a GPU)."""
    from facodec_b200 import build
    return build.build()


# case table shared with oracle/make_golden.py (kept in sync by test_oracle.py::test_case_table)
GOLDEN_CASES = {
    "b2_t7200": dict(wseed=0, xseed=114514, B=2, T=7200, n_c=2),
    "b1_t96000": dict(wseed=0, xseed=114514, B=1, T=96000, n_c=2),
    "b1_t7000_ragged": dict(wseed=0, xseed=7, B=1, T=7000, n_c=2),
    "b3_t1500_short": dict(wseed=1, xseed=9, B=3, T=1500, n_c=1),
    "b2_t6000_fullwaves": dict(wseed=1, xseed=11, B=2, T=6000, n_c=2, full=9000, lens=(9000, 4800)),
}


# voice-conversion fixtures (kept in sync with oracle/make_golden.py by test_oracle.py::test_redecoder_case_table)
REDEC_CASES = {
    "redec_b2_t7200_vc": dict(src="b2_t7200", wseed=0, use_p=False, n_c=1),
    "redec_b2_t7200_full": dict(src="b2_t7200", wseed=0, use_p=True, n_c=2),
    "redec_b3_t1500_short": dict(src="b3_t1500_short", wseed=1, use_p=True, n_c=1),
}


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))


_SD_CACHE = {}


def state_dicts(seed):
    from facodec_b200 import synth
    if seed not in _SD_CACHE:
        _SD_CACHE.clear()
        _SD_CACHE[seed] = synth.synth_state_dicts(seed)
    return _SD_CACHE[seed]


def case_inputs(c):
    from facodec_b200 import synth
    x = synth.synth_waves(c["B"], c["T"], seed=c["xseed"])
    kw = {}
    if "full" in c:
        kw["full_waves"] = synth.synth_waves(c["B"], c["full"], seed=c["xseed"] + 1).squeeze(1)
        kw["wave_lens"] = torch.tensor(c["lens"], dtype=torch.int64)
    return x, kw
