"""TEST INFRASTRUCTURE ONLY — small DSP restatements of third-party helpers the reference calls.

librosa 0.9.1 (requirements.txt) is not installed and not in the reference repository: these follow
its published algorithms; PARITY UNPINNED against the real librosa.
"""
from __future__ import annotations

import numpy as np


def hz_to_mel_htk(f):
    return 2595.0 * np.log10(1.0 + np.asarray(f, dtype=np.float64) / 700.0)


def mel_to_hz_htk(m):
    return 700.0 * (10.0 ** (np.asarray(m, dtype=np.float64) / 2595.0) - 1.0)


def mel_filterbank(sr, n_fft, n_mels=128, fmin=0.0, fmax=None):
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, htk=True, norm='slaney') as called at rmvpe.py:277-284."""
    if fmax is None:
        fmax = sr / 2.0
    n_bins = 1 + n_fft // 2
    fftfreqs = np.linspace(0, sr / 2.0, n_bins)
    mel_f = mel_to_hz_htk(np.linspace(hz_to_mel_htk(fmin), hz_to_mel_htk(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    weights = np.zeros((n_mels, n_bins), dtype=np.float64)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, None]
    return weights.astype(np.float32)


def librosa_rms(y, frame_length, hop_length):
    """librosa.feature.rms(y=..., frame_length, hop_length) of librosa 0.9.1 (center=True, reflect pad),
    as called at vc_infer_pipeline.py:43-46. Returns [1, n_frames]."""
    y = np.asarray(y)
    pad = frame_length // 2
    yp = np.pad(y, (pad, pad), mode="reflect")
    n_frames = 1 + (len(yp) - frame_length) // hop_length
    idx = np.arange(frame_length)[:, None] + hop_length * np.arange(n_frames)[None, :]
    x = yp[idx]
    power = np.mean(np.abs(x) ** 2, axis=0, keepdims=True)
    return np.sqrt(power)


def resample_sinc_mono(x, n_out, rate_in, rate_out, zero_crossings=16):
    """Checker for the device INGEST STAND-IN b200vc_resample_sinc_mono (the reference shells out to ffmpeg
    `-ac 1 -ar 16000`, my_utils.py:13-17 — not restated): channel mean, Hann-windowed sinc, cutoff at the lower Nyquist.
    float64 accumulation; x [channels, n_in] -> [n_out]."""
    x = np.asarray(x, dtype=np.float64)
    mono = x.mean(0)
    n_in = mono.shape[0]
    ratio = float(rate_in) / float(rate_out)
    scale = 1.0 / ratio if ratio > 1.0 else 1.0
    halfw = zero_crossings / scale
    out = np.zeros(n_out)
    kk = np.arange(-int(np.ceil(halfw)) - 1, int(np.ceil(halfw)) + 2)
    for s in range(0, n_out, 65536):
        m = np.arange(s, min(s + 65536, n_out))
        center = m * ratio
        k = np.floor(center)[:, None].astype(np.int64) + kk[None, :]
        d = k - center[:, None]
        ok = (np.abs(d) <= halfw) & (k >= 0) & (k < n_in)
        a = d * scale
        sinc = np.sinc(a)
        win = 0.5 + 0.5 * np.cos(np.pi * d / halfw)
        v = mono[np.clip(k, 0, n_in - 1)]
        out[m] = (np.where(ok, v * sinc * win, 0.0)).sum(1) * scale
    return out.astype(np.float32)


def pcm16_soundfile(x: np.ndarray) -> np.ndarray:
    """`soundfile.write(path, float_array, sr)` to a .wav (default subtype PCM_16; mdx.py:273,280): python-soundfile enables
    libsndfile's clipping for every file it opens (`sf_command(SFC_SET_CLIPPING, SF_TRUE)`), so floats are converted by
    pcm.c f2s_clip_array: scaled = x * (8.0 * 0x10000000) in float; >= 0x7FFFFFFF -> 0x7FFF; <= -8.0 * 0x10000000 -> 0x8000;
    else lrintf(scaled) >> 16.  soundfile / libsndfile are absent from the reference repository: restated from
    their published sources, PARITY UNPINNED."""
    s = np.asarray(x, dtype=np.float32) * np.float32(8.0 * 0x10000000)
    out = np.empty(s.shape, dtype=np.int16)
    flat, o = s.reshape(-1), out.reshape(-1)
    hi, lo = flat >= np.float32(1.0 * 0x7FFFFFFF), flat <= np.float32(-8.0 * 0x10000000)
    mid = ~(hi | lo)
    o[hi], o[lo] = 0x7FFF, -0x8000
    o[mid] = (np.rint(flat[mid]).astype(np.int64) >> 16).astype(np.int16)
    return out
