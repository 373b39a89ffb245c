"""TEST INFRASTRUCTURE -- never imported by the product path.

Imports the *unmodified* reference hot-path modules from a checkout of the reference project
(``$ALDM_REFERENCE_ROOT``, default ``oracle/_ref``, git-ignored) with the package ``__init__``
files bypassed (``audioldm2/__init__.py`` pulls in soundfile, progressbar, phonemizer ... which
are not installed; SURVEY.md 8c).  Used by ``tests/golden/make_golden.py`` to generate the
committed fixtures; no test needs it.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

REF_ROOT = os.environ.get("ALDM_REFERENCE_ROOT") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "audioldm2"))


def _stub_pkg(name: str, path: str):
    if name in sys.modules:
        return
    m = types.ModuleType(name)
    m.__path__ = [path]
    sys.modules[name] = m


def _stub_librosa():
    """stft.py needs three librosa symbols (pad_center, tiny, filters.mel); librosa 0.9.2 is
    not installed.  Supply restatements so the reference STFT/TacotronSTFT classes import.
    The mel basis comes from oracle.mel (Slaney scale + Slaney norm = librosa 0.9.2 defaults)."""
    if "librosa" in sys.modules:
        return
    import numpy as np
    from . import mel as _mel

    lib = types.ModuleType("librosa")
    util = types.ModuleType("librosa.util")
    filt = types.ModuleType("librosa.filters")

    def pad_center(data, size, axis=-1, **kw):
        n = data.shape[axis]
        lpad = int((size - n) // 2)
        lengths = [(0, 0)] * data.ndim
        lengths[axis] = (lpad, int(size - n - lpad))
        return np.pad(data, lengths, **kw)

    def tiny(x):
        x = np.asarray(x)
        dt = x.dtype if np.issubdtype(x.dtype, np.floating) else np.dtype(np.float32)
        return np.finfo(dt).tiny

    def mel(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, **kw):
        return _mel.mel_filterbank(sr, n_fft, n_mels, fmin, fmax)

    util.pad_center = pad_center
    util.tiny = tiny
    util.normalize = lambda x, **kw: x
    filt.mel = mel
    lib.util = util
    lib.filters = filt
    lib.stft = None
    lib.istft = None
    sys.modules["librosa"] = lib
    sys.modules["librosa.util"] = util
    sys.modules["librosa.filters"] = filt


def load():
    """Return a namespace with the reference classes of the hot path."""
    if not available():
        raise RuntimeError(f"reference tree not found at {REF_ROOT}")
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    base = os.path.join(REF_ROOT, "audioldm2")
    _stub_pkg("audioldm2", base)
    _stub_pkg("audioldm2.utilities", os.path.join(base, "utilities"))
    _stub_pkg("audioldm2.utilities.audio", os.path.join(base, "utilities", "audio"))
    _stub_pkg("audioldm2.latent_diffusion", os.path.join(base, "latent_diffusion"))
    _stub_pkg("audioldm2.latent_diffusion.models", os.path.join(base, "latent_diffusion", "models"))
    _stub_pkg("audioldm2.latent_diffusion.modules", os.path.join(base, "latent_diffusion", "modules"))
    ns = types.SimpleNamespace()
    om = importlib.import_module("audioldm2.latent_diffusion.modules.diffusionmodules.openaimodel")
    vm = importlib.import_module("audioldm2.latent_diffusion.modules.diffusionmodules.model")
    ut = importlib.import_module("audioldm2.latent_diffusion.modules.diffusionmodules.util")
    dd = importlib.import_module("audioldm2.latent_diffusion.models.ddim")
    hg = importlib.import_module("audioldm2.hifigan.models")
    ns.UNetModel = om.UNetModel
    ns.Decoder, ns.Encoder = vm.Decoder, vm.Encoder
    ns.DDIMSampler = dd.DDIMSampler
    ns.Generator = hg.Generator
    ns.util = ut
    try:
        _stub_librosa()
        st = importlib.import_module("audioldm2.utilities.audio.stft")
        ns.TacotronSTFT = st.TacotronSTFT
    except Exception as e:  # pragma: no cover
        ns.TacotronSTFT = None
        ns.stft_error = repr(e)
    return ns
