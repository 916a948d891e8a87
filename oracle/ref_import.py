"""TEST INFRASTRUCTURE ONLY — import the *unmodified* reference modules from a checkout of the reference repository
named by the environment variable AICOVERGEN_REFERENCE.

It is how tests/golden/*.npz, which pin the oracle restatements in this directory, are generated
(tools/make_golden.py); the tests themselves only read those files.  Recipe follows SURVEY.md Appendix B10: third-party modules that are
not installed (faiss, librosa, parselmouth, pyworld, torchcrepe, onnxruntime, soundfile,
fairseq) are replaced by inert stubs; nothing of the reference's own arithmetic is touched.
"""
from __future__ import annotations

import importlib
import importlib.machinery
import os
import sys
import types

import numpy as np

REF_ROOT = os.environ.get("AICOVERGEN_REFERENCE", "")
REF_SRC = os.path.join(REF_ROOT, "src")


def available() -> bool:
    return bool(REF_ROOT) and os.path.isdir(REF_SRC)


def _stub(name: str, **attrs):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def _mel_filterbank(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False, norm="slaney", dtype=np.float32):
    from oracle.dsp import mel_filterbank
    assert htk, "only the htk=True variant (rmvpe.py:277-284) is restated"
    return mel_filterbank(sr, n_fft, n_mels, fmin, fmax).astype(dtype)


def _rms(y, frame_length=2048, hop_length=512, center=True, pad_mode="reflect"):
    from oracle.dsp import librosa_rms
    return librosa_rms(y, frame_length, hop_length)


_done = False


def setup():
    """Install stubs and put the reference's src/ on sys.path (idempotent)."""
    global _done
    if _done:
        return
    if not available():
        raise RuntimeError("set AICOVERGEN_REFERENCE to a checkout of the reference repository")
    if not hasattr(np, "int"):
        np.int = int  # vc_infer_pipeline.py:368 uses the removed alias
    import transformers  # noqa: F401  (must be imported before librosa is stubbed: it probes it via find_spec)

    class _NotAvailable:
        def __init__(self, *a, **k):
            raise RuntimeError("third-party module stubbed in oracle/ref_import.py")

    if "faiss" not in sys.modules:
        _stub("faiss", read_index=_NotAvailable)
    if "librosa" not in sys.modules:
        lib = _stub("librosa")
        lib.filters = _stub("librosa.filters", mel=_mel_filterbank)
        lib.feature = _stub("librosa.feature", rms=_rms)
        lib.load = _NotAvailable
        lib.resample = _NotAvailable
    for name in ("parselmouth", "pyworld", "torchcrepe", "soundfile"):
        if name not in sys.modules:
            _stub(name)
    if "onnxruntime" not in sys.modules:
        _stub("onnxruntime", InferenceSession=_NotAvailable)
    if "fairseq" not in sys.modules:
        fs = _stub("fairseq")
        fs.checkpoint_utils = _stub("fairseq.checkpoint_utils", load_model_ensemble_and_task=_NotAvailable)
    if REF_SRC not in sys.path:
        sys.path.insert(0, REF_SRC)
    _done = True


def module(name: str):
    """Import a reference module by its in-repo name, e.g. 'infer_pack.models', 'rmvpe', 'vc_infer_pipeline', 'mdx'."""
    setup()
    return importlib.import_module(name)
