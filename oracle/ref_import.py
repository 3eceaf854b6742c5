"""Import the UNMODIFIED reference model files behind three stub modules (SURVEY.md section 8(c)).

`import olmoasr` fails in this container (openai-whisper is absent and cannot be installed), but
olmoasr/model.py and olmoasr/inf_model.py only need `whisper.decoding.{decode,detect_language}` and
`olmoasr.transcribe.transcribe` as attributes at import time.  The reference checkout (OLMOASR_REFERENCE_ROOT) is
only needed where golden data is generated: everything here is used to VALIDATE oracle/model.py and to GENERATE tests/golden/*, never at
run time on the GPU box.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("OLMOASR_REFERENCE_ROOT", "")   # a checkout of allenai/OLMoASR


def available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isfile(os.path.join(REFERENCE_ROOT, "olmoasr", "model.py"))


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    return m


def load():
    """Returns (ref_model_module, ref_inf_model_module, ref_model_dims_module)."""
    if not available():
        raise RuntimeError(f"reference tree not found under {REFERENCE_ROOT}")
    saved = {k: sys.modules.get(k) for k in ("whisper", "whisper.decoding", "olmoasr", "olmoasr.transcribe",
                                              "olmoasr.model", "olmoasr.inf_model", "olmoasr.config",
                                              "olmoasr.config.model_dims")}
    try:
        def _na(*a, **k):
            raise NotImplementedError("third-party whisper is not installed")

        sys.modules["whisper"] = _stub("whisper")
        sys.modules["whisper.decoding"] = _stub("whisper.decoding", decode=_na, detect_language=_na)
        pkg = _stub("olmoasr")
        pkg.__path__ = [os.path.join(REFERENCE_ROOT, "olmoasr")]
        sys.modules["olmoasr"] = pkg
        sys.modules["olmoasr.transcribe"] = _stub("olmoasr.transcribe", transcribe=_na)
        for k in ("olmoasr.model", "olmoasr.inf_model", "olmoasr.config", "olmoasr.config.model_dims"):
            sys.modules.pop(k, None)
        ref_model = importlib.import_module("olmoasr.model")
        ref_inf = importlib.import_module("olmoasr.inf_model")
        ref_dims = importlib.import_module("olmoasr.config.model_dims")
        return ref_model, ref_inf, ref_dims
    finally:
        # leave no trace: the product package must never resolve `olmoasr` to the reference tree
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
