"""TEST INFRASTRUCTURE ONLY -- imports the *unmodified* reference from FACODEC_REFERENCE_ROOT.

Only usable where the reference tree is present; tests use the fixtures oracle/make_golden.py made from it.
It is used to (1) validate the restatement in ``oracle/facodec_oracle.py``
bit-for-bit and (2) generate the committed fixtures under ``tests/golden/``
(``oracle/make_golden.py``).

Three third-party modules the reference imports are not installed here and
carry no arithmetic on the encode->quantize->decode path; they are replaced by
placeholder modules (SURVEY.md section 8c):

* ``audiotools`` -- imported at dac/__init__.py:6-9, dac/model/dac.py:7-8,
  dac/model/base.py:9, dac/model/discriminator.py:4-6, dac/nn/loss.py:6-7.
* ``munch``      -- modules/commons.py:6 (attribute dict).
* ``argbind``    -- dac/utils/__init__.py:3-9 (decorator).
"""
import os
import sys
import types

import torch
from torch import nn

REFERENCE_ROOT = os.environ.get("FACODEC_REFERENCE_ROOT", "")   # the reference tree, when present


class _Anything(types.ModuleType):
    """Module whose every attribute resolves to a harmless placeholder."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        sub = _Placeholder(name)
        setattr(self, name, sub)
        return sub


class _Placeholder:
    def __init__(self, name="placeholder"):
        self._name = name

    def __call__(self, *a, **k):
        # used as decorator (argbind.bind(...)) or as a constructor
        if len(a) == 1 and callable(a[0]) and not k:
            return a[0]
        return _Placeholder(self._name)

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Placeholder(name)

    def __mro_entries__(self, bases):
        return (object,)


class Munch(dict):
    """6-line stand-in for munch.Munch (dict with attribute access)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


def _install_stubs():
    if "audiotools" not in sys.modules:
        at = _Anything("audiotools")
        ml = _Anything("audiotools.ml")

        class BaseModel(nn.Module):
            INTERN = []
            EXTERN = []

        ml.BaseModel = BaseModel
        at.ml = ml
        at.AudioSignal = _Placeholder("AudioSignal")
        at.STFTParams = _Placeholder("STFTParams")
        sys.modules["audiotools"] = at
        sys.modules["audiotools.ml"] = ml
        for sub in ("core", "data", "metrics"):
            m = _Anything("audiotools." + sub)
            setattr(at, sub, m)
            sys.modules["audiotools." + sub] = m
    if "munch" not in sys.modules:
        m = types.ModuleType("munch")
        m.Munch = Munch
        sys.modules["munch"] = m
    for name in ("soundfile", "librosa"):      # meldataset.py:8-9 (file I/O only; PseudoDataset never calls them)
        if name not in sys.modules:
            sys.modules[name] = _Anything(name)
    if "argbind" not in sys.modules:
        ab = _Anything("argbind")
        ab.bind = lambda *a, **k: (a[0] if (len(a) == 1 and callable(a[0]) and not k) else (lambda f: f))
        sys.modules["argbind"] = ab


def available():
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "dac"))


def recursive_munch(d):
    # same behaviour as modules/commons.py:473-479
    if isinstance(d, dict):
        return Munch((k, recursive_munch(v)) for k, v in d.items())
    if isinstance(d, list):
        return [recursive_munch(v) for v in d]
    return d


def import_reference():
    """Returns the reference's modules/commons module (build_model lives there)."""
    if not available():
        raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
    _install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import modules.commons as commons  # noqa
    return commons


def build_reference_redecoder(seed=0):
    """build_model(config_redecoder.yml model_params, stage='redecoder') as reconstruct_redecoder.py:43-61 does:
    Munch(encoder=Redecoder (wavenet), decoder=Decoder(causal=False, lstm=0)), eval mode, CPU fp32."""
    import yaml
    commons = import_reference()
    cfg = yaml.safe_load(open(os.path.join(REFERENCE_ROOT, "configs", "config_redecoder.yml")))
    params = recursive_munch(cfg["model_params"])
    torch.manual_seed(seed)
    model = commons.build_model(params, stage="redecoder")
    out = Munch(encoder=model.encoder, decoder=model.decoder)
    for k in out:
        out[k].eval()
    return out


def build_reference_model(seed=0):
    """build_model(config.yml model_params) exactly as reconstruct.py:19-37 does,
    restricted to the three hot-path modules, eval mode, CPU fp32."""
    import yaml
    commons = import_reference()
    cfg = yaml.safe_load(open(os.path.join(REFERENCE_ROOT, "configs", "config.yml")))
    params = recursive_munch(cfg["model_params"])
    torch.manual_seed(seed)
    model = commons.build_model(params, stage="codec")
    out = Munch(encoder=model.encoder, quantizer=model.quantizer, decoder=model.decoder)
    for k in out:
        out[k].eval()
    return out
