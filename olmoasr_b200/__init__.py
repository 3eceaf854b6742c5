"""olmoasr_b200 -- H100-native (sm_90a) implementation of the OLMoASR training / decode hot path behind the
reference's Python surface (olmoasr/__init__.py): `load_model`, `model`, `inf_model`, `log_mel_spectrogram`,
`pad_or_trim`, `load_audio`.  See README.md for scope and INTEGRATION.md for how to swap it in."""
import io
import os
from typing import Optional, Union

import torch

from . import inf_model, model
from .audio import load_audio, log_mel_spectrogram, pad_or_trim
from .config.model_dims import VARIANT_TO_DIMS, ModelDimensions

__all__ = ["load_model", "model", "inf_model", "load_audio", "log_mel_spectrogram", "pad_or_trim", "ModelDimensions",
           "VARIANT_TO_DIMS"]


def load_model(name: str, device: Optional[Union[str, torch.device]] = None, download_root: Optional[str] = None,
               inference: bool = False, in_memory: bool = False):
    """Load a checkpoint written by the reference (olmoasr/__init__.py:97-166): a dict with "dims" (dict or
    ModelDimensions) and "model_state_dict".  `name` must be a local file: this package has no download table (the
    HF-hub fetch of the reference, __init__.py:33-93, is control plane and out of scope)."""
    if device is None:
        device = "cuda" if torch.cuda.is_available() else "cpu"
    if not os.path.isfile(name):
        raise ValueError(f"Model '{name}' not found: pass the path of a checkpoint file "
                         "(model identifiers are resolved by the reference's downloader, which is not part of this package)")
    if in_memory:
        with open(name, "rb") as f:
            blob = f.read()
        fp = io.BytesIO(blob)
    else:
        fp = open(name, "rb")
    with fp:
        checkpoint = torch.load(fp, map_location=device, weights_only=False)
    dims = checkpoint["dims"]
    if not isinstance(dims, dict):
        dims = dict(vars(dims))
    dims = ModelDimensions(**dims)
    state = checkpoint["model_state_dict"]
    state = {k[len("module."):] if k.startswith("module.") else k: v for k, v in state.items()}  # *_ddp.pt checkpoints
    instance = inf_model.OLMoASR(dims) if inference else model.OLMoASR(dims)
    instance.load_state_dict(state)
    return instance.to(device)
