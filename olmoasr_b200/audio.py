"""GPU log-mel front end with the upstream whisper.audio API (olmoasr/__init__.py:21 re-exports
`load_audio, log_mel_spectrogram, pad_or_trim`; call sites: scripts/training/train_timestamps.py:196-214,
scripts/eval/eval.py:157-162, olmoasr/transcribe.py:148).

`log_mel_spectrogram` here takes a waveform or a BATCH of waveforms that is (or is moved) on a CUDA device and
runs the fused sm_90a kernel (csrc/logmel.cu).  The dynamic-range floor uses each clip's own maximum -- the
per-sample semantics of the reference datasets.  There is no CPU implementation in this package.
"""
from __future__ import annotations

import math
from functools import lru_cache
from typing import Optional, Union

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from ._lib import call, ptr, stream

SAMPLE_RATE = 16000
N_FFT = 400
HOP_LENGTH = 160
CHUNK_LENGTH = 30
N_SAMPLES = CHUNK_LENGTH * SAMPLE_RATE  # 480000 samples in a 30-second chunk
N_FRAMES = N_SAMPLES // HOP_LENGTH  # 3000 frames in a mel spectrogram input
N_SAMPLES_PER_TOKEN = HOP_LENGTH * 2
FRAMES_PER_SECOND = SAMPLE_RATE // HOP_LENGTH
TOKENS_PER_SECOND = SAMPLE_RATE // N_SAMPLES_PER_TOKEN


def pad_or_trim(array, length: int = N_SAMPLES, *, axis: int = -1):
    """Pad or trim the audio array to `length` samples along `axis` (torch tensors or numpy arrays)."""
    if torch.is_tensor(array):
        if array.shape[axis] > length:
            array = array.index_select(dim=axis, index=torch.arange(length, device=array.device))
        if array.shape[axis] < length:
            pad_widths = [(0, 0)] * array.ndim
            pad_widths[axis] = (0, length - array.shape[axis])
            array = F.pad(array, [p for sizes in pad_widths[::-1] for p in sizes])
    else:
        if array.shape[axis] > length:
            array = array.take(indices=range(length), axis=axis)
        if array.shape[axis] < length:
            pad_widths = [(0, 0)] * array.ndim
            pad_widths[axis] = (0, length - array.shape[axis])
            array = np.pad(array, pad_widths)
    return array


def load_audio(file: str, sr: int = SAMPLE_RATE):
    """Decode an audio file to mono float32 at `sr` via the ffmpeg CLI (same contract as whisper.audio.load_audio)."""
    from subprocess import CalledProcessError, run

    cmd = ["ffmpeg", "-nostdin", "-threads", "0", "-i", file, "-f", "s16le", "-ac", "1", "-acodec", "pcm_s16le",
           "-ar", str(sr), "-"]
    try:
        out = run(cmd, capture_output=True, check=True).stdout
    except (CalledProcessError, FileNotFoundError) as e:
        raise RuntimeError(f"Failed to load audio: {getattr(e, 'stderr', e)}") from e
    return np.frombuffer(out, np.int16).flatten().astype(np.float32) / 32768.0


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    logstep = math.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_hz / f_sp + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(n_mels: int = 80) -> np.ndarray:
    """Slaney-scale, slaney-normalised triangular filterbank (n_mels, 201) f32: what upstream ships as
    assets/mel_filters.npz (= librosa.filters.mel(sr=16000, n_fft=400, n_mels=n_mels))."""
    assert n_mels in (80, 128), f"Unsupported n_mels: {n_mels}"
    fft_f = np.linspace(0.0, SAMPLE_RATE / 2.0, 1 + N_FFT // 2)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(SAMPLE_RATE / 2.0), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fft_f[None, :]
    w = np.maximum(0.0, np.minimum(-ramps[:-2] / fdiff[:-1, None], ramps[2:] / fdiff[1:, None]))
    w *= (2.0 / (mel_f[2: n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w.astype(np.float32)


@lru_cache(maxsize=8)
def _device_tables(device_index: int, n_mels: int):
    dev = torch.device("cuda", device_index)
    n = np.arange(N_FFT, dtype=np.float64)
    window = (0.5 - 0.5 * np.cos(2.0 * np.pi * n / N_FFT)).astype(np.float32)  # torch.hann_window(400) (periodic)
    cos_t = np.cos(2.0 * np.pi * n / N_FFT).astype(np.float32)
    sin_t = np.sin(2.0 * np.pi * n / N_FFT).astype(np.float32)
    filt = mel_filterbank(n_mels)
    nz = filt != 0
    klo = np.array([int(np.argmax(r)) if r.any() else 0 for r in nz], dtype=np.int32)
    khi = np.array([int(len(r) - np.argmax(r[::-1])) if r.any() else 0 for r in nz], dtype=np.int32)
    t = lambda a: torch.from_numpy(a).to(dev)
    return t(window), t(cos_t), t(sin_t), t(filt), t(klo), t(khi)


def log_mel_spectrogram(audio: Union[str, np.ndarray, torch.Tensor], n_mels: int = 80, padding: int = 0,
                        device: Optional[Union[str, torch.device]] = None) -> torch.Tensor:
    """Log-mel spectrogram of a waveform (n,) or batch (B, n): float32 or int16 samples at 16 kHz.

    Returns (n_mels, n // 160) or (B, n_mels, n // 160) float32 on the CUDA device, n = samples + padding, any length
    >= 400 (upstream: n // 160 frames for every n).  Rows are padded to whole 640-sample groups for the kernel, which is
    told the true length: the end reflection of torch.stft happens there, padded frames are dropped."""
    if not torch.is_tensor(audio):
        if isinstance(audio, str):
            audio = load_audio(audio)
        audio = torch.from_numpy(np.ascontiguousarray(audio))
    if device is not None:
        audio = audio.to(device)
    if not audio.is_cuda:
        if not torch.cuda.is_available():
            raise _lib.OasrError("log_mel_spectrogram runs on the GPU only (no CPU fallback); no CUDA device is visible")
        audio = audio.cuda()
    squeeze = audio.dim() == 1
    if squeeze:
        audio = audio[None]
    if audio.dim() != 2:
        raise ValueError(f"audio must be (n,) or (B, n), got {tuple(audio.shape)}")
    if audio.dtype not in (torch.float32, torch.int16):
        audio = audio.float()
    if padding > 0:
        audio = F.pad(audio, (0, padding))
    n_true = audio.shape[1]
    if n_true < N_FFT:
        raise ValueError(f"need at least {N_FFT} samples, got {n_true}")
    group = 4 * HOP_LENGTH
    if n_true % group != 0:
        audio = F.pad(audio, (0, group - n_true % group))
    audio = audio.contiguous()
    B, n = audio.shape
    window, cos_t, sin_t, filt, klo, khi = _device_tables(audio.device.index or 0, n_mels)
    out = torch.empty((B, n_mels, n // HOP_LENGTH), device=audio.device, dtype=torch.float32)
    clip_max = torch.empty(B, device=audio.device, dtype=torch.float32)
    call("oasr_logmel", ptr(audio), int(audio.dtype == torch.int16), ptr(window), ptr(cos_t), ptr(sin_t), ptr(filt),
         ptr(klo), ptr(khi), ptr(out), ptr(clip_max), B, n, n_mels, n_true, stream())
    if n != n_true:
        out = out[:, :, : n_true // HOP_LENGTH]
    return out[0] if squeeze else out
