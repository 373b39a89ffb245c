"""TEST INFRASTRUCTURE -- CPU restatement of the STFT / mel front end (SURVEY.md 8a row A12).

PARITY UNPINNED for the mel filterbank: the arithmetic lives in the third-party dependency
``librosa==0.9.2`` (pinned in the reference's setup.py:48, not vendored in the reference,
not installed here).  ``mel_filterbank`` restates librosa 0.9.2's published algorithm
(``librosa.filters.mel`` with its defaults ``htk=False, norm="slaney"``), which is what the
reference call site ``librosa_mel_fn(sampling_rate, filter_length, n_mel_channels, mel_fmin,
mel_fmax)`` (utilities/audio/stft.py:145-147) evaluates.  No reference test holds a golden
vector for it.

The STFT part *is* pinned: ``stft_mel`` is checked against the reference ``TacotronSTFT``
class (imported with this filterbank injected) by tests/golden/make_golden.py, and against
``torch.stft`` in tests/test_oracle.py.
"""
from __future__ import annotations

import numpy as np


def _hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    big = f >= min_log_hz
    out = mels.copy()
    out[big] = min_log_mel + np.log(f[big] / min_log_hz) / logstep
    return out


def _mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    freqs = f_sp * m
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    big = m >= min_log_mel
    freqs[big] = min_log_hz * np.exp(logstep * (m[big] - min_log_mel))
    return freqs


def mel_filterbank(sr, n_fft, n_mels, fmin=0.0, fmax=None) -> np.ndarray:
    """Slaney-scale triangular filters with Slaney area normalisation -> float32 [n_mels, 1+n_fft//2]."""
    if fmax is None:
        fmax = sr / 2.0
    n_bins = 1 + n_fft // 2
    fftfreqs = np.linspace(0.0, sr / 2.0, n_bins)
    mel_pts = np.linspace(_hz_to_mel(np.array([fmin]))[0], _hz_to_mel(np.array([fmax]))[0], n_mels + 2)
    mel_f = _mel_to_hz(mel_pts)
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((n_mels, n_bins), dtype=np.float64)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    w *= enorm[:, None]
    return w.astype(np.float32)


def hann_periodic(n: int) -> np.ndarray:
    """scipy.signal.get_window("hann", n, fftbins=True) (stft.py:41)."""
    return (0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n) / n)).astype(np.float64)


def stft_mel(wav: np.ndarray, n_fft: int, hop: int, n_mels: int, sr: int, fmin: float, fmax: float,
             clip_val: float = 1e-5):
    """``TacotronSTFT.mel_spectrogram`` (stft.py:159-178) for wav [B, T] -> (log-mel [B, n_mels, frames],
    magnitude [B, bins, frames]); win_length == filter_length as in every reference config.

    Follows STFT.transform (stft.py:52-81): reflect-pad n_fft/2 both sides, frame with stride
    ``hop``, multiply by the periodic Hann window, real DFT, magnitude; then mel_basis @ mag and
    log(clamp(., 1e-5)) (audio_processing.py:85-91).  Evaluated in float64, returned as float32.
    """
    wav = np.asarray(wav, dtype=np.float64)
    B, T = wav.shape
    pad = n_fft // 2
    x = np.pad(wav, ((0, 0), (pad, pad)), mode="reflect")
    n_frames = (x.shape[1] - n_fft) // hop + 1
    idx = np.arange(n_fft)[None, :] + hop * np.arange(n_frames)[:, None]
    frames = x[:, idx] * hann_periodic(n_fft)[None, None, :]
    spec = np.fft.rfft(frames, axis=-1)                       # [B, frames, bins]
    mag = np.abs(spec).transpose(0, 2, 1)                     # [B, bins, frames]
    basis = mel_filterbank(sr, n_fft, n_mels, fmin, fmax).astype(np.float64)
    mel = np.einsum("mk,bkt->bmt", basis, mag)
    logmel = np.log(np.maximum(mel, clip_val))
    return logmel.astype(np.float32), mag.astype(np.float32)
