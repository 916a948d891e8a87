"""TEST INFRASTRUCTURE ONLY — CPU restatement of the MDX-Net separation pass (src/mdx.py).

* `stft` / `istft`, `segment`, `pad_wave`, `process_wave`, the `run_mdx` arithmetic: follow mdx.py:19-54,
  92-235, 257-280 and are pinned against the reference's own classes (tests/test_oracle_vs_reference.py).
* `convtdfnet`: the TFC-TDF U-Net that lives inside the UVR-MDX-NET `.onnx` files (mdx.py:74-77,
  download_models.py:23-26).  The ONNX graphs are not in the reference repository and onnxruntime is not installed:
  restated from the public KUIELab / UVR "ConvTDFNet" architecture (SURVEY.md §8(c)); PARITY UNPINNED.
"""
from __future__ import annotations

from typing import Callable, Dict

import numpy as np
import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]
BN_EPS = 1e-5


class MdxParams:
    """MDXModel.__init__ (mdx.py:19-35)."""

    def __init__(self, dim_f, dim_t, n_fft, hop=1024, stem_name=None, compensation=1.0):
        self.dim_f, self.dim_t, self.dim_c, self.n_fft, self.hop = dim_f, dim_t, 4, n_fft, hop
        self.stem_name, self.compensation = stem_name, compensation
        self.n_bins = n_fft // 2 + 1
        self.chunk_size = hop * (dim_t - 1)
        self.window = torch.hann_window(window_length=n_fft, periodic=True)

    def stft(self, x):
        """mdx.py:37-43: [B,2,chunk] -> [B,4,dim_f,dim_t] (channels L.re, L.im, R.re, R.im)."""
        x = x.reshape([-1, self.chunk_size])
        x = torch.stft(x, n_fft=self.n_fft, hop_length=self.hop, window=self.window, center=True, return_complex=True)
        x = torch.view_as_real(x).permute([0, 3, 1, 2])
        x = x.reshape([-1, 2, 2, self.n_bins, self.dim_t]).reshape([-1, 4, self.n_bins, self.dim_t])
        return x[:, :, :self.dim_f]

    def istft(self, x):
        """mdx.py:45-54."""
        pad = torch.zeros([x.shape[0], 4, self.n_bins - self.dim_f, self.dim_t])
        x = torch.cat([x, pad], -2)
        x = x.reshape([-1, 2, 2, self.n_bins, self.dim_t]).reshape([-1, 2, self.n_bins, self.dim_t])
        x = torch.view_as_complex(x.permute([0, 2, 3, 1]).contiguous())
        x = torch.istft(x, n_fft=self.n_fft, hop_length=self.hop, window=self.window, center=True)
        return x.reshape([-1, 2, self.chunk_size])


# ---------------------------------------------------------------------------
# ConvTDFNet (TFC-TDF v2 U-Net)
# ---------------------------------------------------------------------------
def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False, 0.0, BN_EPS)


def _tfc_tdf(sd: SD, p: str, x, l: int):
    for j in range(l):
        x = F.relu(_bn(sd, f"{p}.tfc.H.{j}.1", F.conv2d(x, sd[f"{p}.tfc.H.{j}.0.weight"], sd[f"{p}.tfc.H.{j}.0.bias"], padding=1)))
    t = F.relu(_bn(sd, f"{p}.tdf.1", F.linear(x, sd[f"{p}.tdf.0.weight"])))
    t = F.relu(_bn(sd, f"{p}.tdf.4", F.linear(t, sd[f"{p}.tdf.3.weight"])))
    return x + t


def convtdfnet(sd: SD, x: torch.Tensor) -> torch.Tensor:
    """[B,4,dim_f,dim_t] -> same shape."""
    dim_f, dim_t, g, l, n, bn, k, dim_c = [int(v) for v in sd["_meta"]]
    with torch.no_grad():
        x = F.relu(_bn(sd, "first_conv.1", F.conv2d(x, sd["first_conv.0.weight"], sd["first_conv.0.bias"])))
        x = x.transpose(-1, -2)
        skips = []
        for i in range(n):
            x = _tfc_tdf(sd, f"encoding_blocks.{i}", x, l)
            skips.append(x)
            x = F.relu(_bn(sd, f"ds.{i}.1", F.conv2d(x, sd[f"ds.{i}.0.weight"], sd[f"ds.{i}.0.bias"], stride=2)))
        x = _tfc_tdf(sd, "bottleneck_block", x, l)
        for i in range(n):
            x = F.relu(_bn(sd, f"us.{i}.1", F.conv_transpose2d(x, sd[f"us.{i}.0.weight"], sd[f"us.{i}.0.bias"], stride=2)))
            x = x * skips[-i - 1]
            x = _tfc_tdf(sd, f"decoding_blocks.{i}", x, l)
        x = x.transpose(-1, -2)
        return F.conv2d(x, sd["final_conv.0.weight"], sd["final_conv.0.bias"])


# ---------------------------------------------------------------------------
# chunking (mdx.py:92-235)
# ---------------------------------------------------------------------------
def segment_split(wave: np.ndarray, chunk_size: int, margin_size: int = 44100):
    """MDX.segment(combine=False) (mdx.py:119-141)."""
    out = []
    n = wave.shape[-1]
    if chunk_size <= 0 or chunk_size > n:
        chunk_size = n
    if margin_size > chunk_size:
        margin_size = chunk_size
    for count, skip in enumerate(range(0, n, chunk_size)):
        margin = 0 if count == 0 else margin_size
        end = min(skip + chunk_size + margin_size, n)
        out.append(wave[:, skip - margin:end].copy())
        if end == n:
            break
    return out


def segment_combine(parts, margin_size: int = 44100):
    """MDX.segment(combine=True) (mdx.py:107-117)."""
    res = None
    for i, seg in enumerate(parts):
        start = 0 if i == 0 else margin_size
        end = None if i == len(parts) - 1 else -margin_size
        if margin_size == 0:
            end = None
        res = seg[:, start:end] if res is None else np.concatenate((res, seg[:, start:end]), axis=-1)
    return res


def pad_wave(wave: np.ndarray, mp: MdxParams):
    """MDX.pad_wave (mdx.py:143-171)."""
    n = wave.shape[1]
    trim = mp.n_fft // 2
    gen = mp.chunk_size - 2 * trim
    pad = gen - n % gen
    wp = np.concatenate((np.zeros((2, trim)), wave, np.zeros((2, pad)), np.zeros((2, trim))), 1)
    chunks = [np.array(wp[:, i:i + mp.chunk_size]) for i in range(0, n + pad, gen)]
    return torch.tensor(np.array(chunks), dtype=torch.float32), pad, trim


def process_wave(wave: np.ndarray, mp: MdxParams, net: Callable[[torch.Tensor], torch.Tensor], mt_threads: int = 2):
    """MDX.process_wave + _process_wave (mdx.py:173-235), single-threaded (results are order independent)."""
    chunk = wave.shape[-1] // mt_threads
    waves = segment_split(wave, chunk)
    outs = []
    for batch in waves:
        mix, pad, trim = pad_wave(batch, mp)
        pw = []
        for m in mix.split(1):
            spec = mp.stft(m)
            proc = net(spec)
            w = mp.istft(proc)
            pw.append(w[:, :, trim:-trim].transpose(0, 1).reshape(2, -1).numpy())
        outs.append(np.concatenate(pw, axis=-1)[:, :-pad])
    return segment_combine(outs)


def run_mdx_arrays(wave: np.ndarray, mp: MdxParams, net, denoise: bool = False, m_threads: int = 2):
    """The arithmetic of run_mdx (mdx.py:257-280) on arrays: returns (main_stem, inverse_stem), float arrays [2,N].
    NB the reference peak-normalises `wave` IN PLACE, so the inverse stem mixes the processed stem (rescaled by
    `peak`) with the NORMALISED input (mdx.py:259-260, 280)."""
    wave = wave.copy()
    peak = max(np.max(wave), abs(np.min(wave)))
    wave /= peak
    if denoise:
        proc = -(process_wave(-wave, mp, net, m_threads)) + process_wave(wave, mp, net, m_threads)
        proc *= 0.5
    else:
        proc = process_wave(wave, mp, net, m_threads)
    proc *= peak
    inverse = (-proc.T * mp.compensation) + wave.T
    return proc, inverse.T
