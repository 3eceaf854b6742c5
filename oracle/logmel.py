"""numpy restatement of the log-mel front end the reference calls per sample on the CPU.

Reference call sites: scripts/training/train_timestamps.py:196-214 (int16 -> /32768 -> pad_or_trim ->
log_mel_spectrogram), scripts/eval/eval.py:157-162, olmoasr/transcribe.py:148; re-exported at
olmoasr/__init__.py:21.  The arithmetic lives in openai-whisper `whisper/audio.py` (absent from
the reference checkout); this file restates its published algorithm:

    pad_or_trim(array, 480000)            zero-pad / truncate the last axis
    stft  = torch.stft(audio, 400, 160, window=hann(400), center=True (reflect pad), return_complex)
    mag   = |stft[..., :-1]|**2                                   (201, 3000)
    mel   = mel_filters(80) @ mag         slaney-scale, slaney-norm filterbank == librosa.filters.mel
    x     = log10(clamp(mel, 1e-10)); x = max(x, x.max() - 8); x = (x + 4) / 4

The oracle computes in float64 and returns float32 (the fp32-vs-fp64 self-noise of the reference is
~4e-6, SURVEY.md section 7 step 3).
"""
from __future__ import annotations

import numpy as np

SAMPLE_RATE = 16000
N_FFT = 400
HOP_LENGTH = 160
CHUNK_LENGTH = 30
N_SAMPLES = CHUNK_LENGTH * SAMPLE_RATE  # 480000
N_FRAMES = N_SAMPLES // HOP_LENGTH  # 3000


def pad_or_trim(array: np.ndarray, length: int = N_SAMPLES, axis: int = -1) -> np.ndarray:
    """whisper.audio.pad_or_trim."""
    if array.shape[axis] > length:
        array = array.take(indices=range(length), axis=axis)
    if array.shape[axis] < length:
        pad = [(0, 0)] * array.ndim
        pad[axis] = (0, length - array.shape[axis])
        array = np.pad(array, pad)
    return array


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, mels)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filters(n_mels: int = 80, sr: int = SAMPLE_RATE, n_fft: int = N_FFT) -> np.ndarray:
    """librosa.filters.mel(sr=16000, n_fft=400, n_mels=80) (what whisper ships as assets/mel_filters.npz):
    slaney mel scale, triangular filters, slaney area normalisation.  Returns (n_mels, 1 + n_fft//2) f32."""
    fftfreqs = np.linspace(0.0, sr / 2.0, 1 + n_fft // 2)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(sr / 2.0), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    weights = np.maximum(0.0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2 : n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, None]
    return weights.astype(np.float32)


def hann_window(n: int = N_FFT) -> np.ndarray:
    """torch.hann_window(n) (periodic)."""
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n) / n)


def stft_power(audio: np.ndarray) -> np.ndarray:
    """|STFT|^2 with torch.stft(center=True, pad_mode='reflect') framing, last frame dropped.
    audio (..., n) -> (..., 201, n // 160)."""
    audio = np.asarray(audio, dtype=np.float64)
    pad = N_FFT // 2
    x = np.pad(audio, [(0, 0)] * (audio.ndim - 1) + [(pad, pad)], mode="reflect")
    n_frames = 1 + (x.shape[-1] - N_FFT) // HOP_LENGTH
    idx = np.arange(N_FFT)[None, :] + HOP_LENGTH * np.arange(n_frames)[:, None]
    frames = x[..., idx] * hann_window()
    spec = np.fft.rfft(frames, n=N_FFT, axis=-1)  # (..., frames, 201)
    power = spec.real**2 + spec.imag**2
    return np.swapaxes(power, -1, -2)[..., :-1]


def log_mel_spectrogram(audio: np.ndarray, n_mels: int = 80, padding: int = 0) -> np.ndarray:
    """whisper.audio.log_mel_spectrogram for one waveform (n,) or a batch (B, n).  The dynamic-range floor
    uses the maximum of EACH waveform's spectrogram: the reference datasets call the function per sample
    (train_timestamps.py:214), so a batched call here means "per-sample", not upstream's whole-tensor max."""
    audio = np.asarray(audio)
    if padding > 0:
        audio = np.pad(audio, [(0, 0)] * (audio.ndim - 1) + [(0, padding)])
    power = stft_power(audio)
    mel = mel_filters(n_mels).astype(np.float64) @ power
    log_spec = np.log10(np.maximum(mel, 1e-10))
    mx = log_spec.max(axis=(-2, -1), keepdims=True)
    log_spec = np.maximum(log_spec, mx - 8.0)
    return ((log_spec + 4.0) / 4.0).astype(np.float32)


def int16_to_float(x: np.ndarray) -> np.ndarray:
    """train_timestamps.py:196 -- np.load(int16).astype(float32) / 32768.0"""
    return x.astype(np.float32) / 32768.0
