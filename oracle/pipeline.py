"""TEST INFRASTRUCTURE ONLY — CPU restatement of `VC.pipeline` (vc_infer_pipeline.py:474-653) composed from the
oracle restatements of its operators (oracle/hubert.py, rmvpe.py, synth.py, index.py).

Pinned against the reference's own `VC.pipeline` run unmodified with duck-typed operators
(tools/make_golden.py, tests/test_oracle_vs_reference.py).  It is also what bench.py times as the CPU
baseline / `--impl reference` arm.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F
from scipy import signal

from . import hubert as ohub
from . import rmvpe as ormv
from . import synth as osyn
from .dsp import librosa_rms
from .index import IvfFlatIndex

bh, ah = signal.butter(N=5, Wn=48, btype="high", fs=16000)      # vc_infer_pipeline.py:22


def change_rms(data1, sr1, data2, sr2, rate):
    """vc_infer_pipeline.py:41-60."""
    rms1 = librosa_rms(data1, sr1 // 2 * 2, sr1 // 2)
    rms2 = librosa_rms(data2, sr2 // 2 * 2, sr2 // 2)
    rms1 = F.interpolate(torch.from_numpy(rms1).unsqueeze(0), size=data2.shape[0], mode="linear").squeeze()
    rms2 = F.interpolate(torch.from_numpy(rms2).unsqueeze(0), size=data2.shape[0], mode="linear").squeeze()
    rms2 = torch.max(rms2, torch.zeros_like(rms2) + 1e-6)
    data2 *= (torch.pow(rms1, torch.tensor(1 - rate)) * torch.pow(rms2, torch.tensor(rate - 1))).numpy()
    return data2


def cut_points(audio: np.ndarray, window=160, t_max=1040000, t_center=960000, t_query=160000):
    """vc_infer_pipeline.py:514-528."""
    audio_pad = np.pad(audio, (window // 2, window // 2), mode="reflect")
    opt_ts = []
    if audio_pad.shape[0] > t_max:
        audio_sum = np.zeros_like(audio)
        for i in range(window):
            audio_sum += audio_pad[i: i - window]
        for t in range(t_center, audio.shape[0], t_center):
            seg = np.abs(audio_sum[t - t_query: t + t_query])
            opt_ts.append(t - t_query + np.where(seg == seg.min())[0][0])
    return opt_ts


def vc_segment(hubert_sd, cpt, audio0, pitch, pitchf, index, big_npy, index_rate, version, protect, window=160):
    """VC.vc (vc_infer_pipeline.py:372-472), fp32. RNG: uses the global torch CPU generator like the reference."""
    feats = torch.from_numpy(audio0).float().view(1, -1)
    feats = ohub.extract_features(hubert_sd, feats, 9 if version == "v1" else 12)
    if version == "v1":
        feats = ohub.final_proj(hubert_sd, feats)
    has_f0 = pitch is not None and pitchf is not None
    if protect < 0.5 and has_f0:
        feats0 = feats.clone()
    if index is not None and big_npy is not None and index_rate != 0:
        npy = feats[0].numpy()
        score, ix = index.search(npy, k=8)
        with np.errstate(divide="ignore", invalid="ignore"):
            weight = np.square(1 / score)
            weight /= weight.sum(axis=1, keepdims=True)
        npy = np.sum(big_npy[ix] * np.expand_dims(weight, axis=2), axis=1)
        feats = torch.from_numpy(npy).unsqueeze(0) * index_rate + (1 - index_rate) * feats
    feats = F.interpolate(feats.permute(0, 2, 1), scale_factor=2).permute(0, 2, 1)
    if protect < 0.5 and has_f0:
        feats0 = F.interpolate(feats0.permute(0, 2, 1), scale_factor=2).permute(0, 2, 1)
    p_len = audio0.shape[0] // window
    if feats.shape[1] < p_len:
        p_len = feats.shape[1]
        if has_f0:
            pitch = pitch[:, :p_len]
            pitchf = pitchf[:, :p_len]
    if protect < 0.5 and has_f0:
        pitchff = pitchf.clone()
        pitchff[pitchf > 0] = 1
        pitchff[pitchf < 1] = protect
        pitchff = pitchff.unsqueeze(-1)
        feats = feats * pitchff + feats0 * (1 - pitchff)
        feats = feats.to(feats0.dtype)
    cfg = cpt["config"]
    upp = int(np.prod(cfg[12]))
    # draw order inside net_g.infer: randn_like(m_p), rand(1,1), randn_like(sine)  (models.py:748,337,368)
    P = feats.shape[1]
    nz = torch.randn(1, cfg[2], P)
    ns = None
    if has_f0:                       # the *_nono models draw randn_like(m_p) only (models.py:847-853)
        _ = torch.rand(1, 1)
        ns = torch.randn(1, P * upp, 1)
    o = osyn.infer(cpt, feats, pitch, pitchf, torch.tensor([0]), nz, ns)
    return o[0, 0].float().numpy()


def pipeline(hubert_sd, cpt, rmvpe_sd, audio: np.ndarray, index: Optional[IvfFlatIndex] = None, f0_up_key=0,
             index_rate=0.5, rms_mix_rate=0.25, protect=0.33, version="v2", x_pad=3, x_query=10, x_center=60,
             x_max=65, seed: Optional[int] = None, return_all=False, if_f0: int = 1):
    """VC.pipeline with f0_method='rmvpe', resample_sr=0, no f0 file (if_f0=0: the no-pitch models, :548-603)."""
    tgt_sr = cpt["config"][-1]
    sr, window = 16000, 160
    t_pad, t_pad_tgt = sr * x_pad, tgt_sr * x_pad
    t_pad2, t_query, t_center, t_max = t_pad * 2, sr * x_query, sr * x_center, sr * x_max
    big_npy = index.reconstruct_n(0, index.ntotal) if (index is not None and index_rate != 0) else None
    if big_npy is None:
        index = None
    audio = signal.filtfilt(bh, ah, audio)
    opt_ts = cut_points(audio, window, t_max, t_center, t_query)
    audio_pad = np.pad(audio, (t_pad, t_pad), mode="reflect")
    p_len = audio_pad.shape[0] // window
    f0 = pitch = pitchf = None
    if if_f0 == 1:
        f0 = ormv.infer_from_audio(rmvpe_sd, audio_pad, 0.03)
        pitch, pitchf = ormv.coarse_pitch(f0, f0_up_key)
        pitch, pitchf = pitch[:p_len], pitchf[:p_len]
        pitch_t = torch.tensor(pitch).unsqueeze(0).long()
        pitchf_t = torch.tensor(pitchf).unsqueeze(0).float()
    sl = (lambda a, b: (pitch_t[:, a:b], pitchf_t[:, a:b])) if if_f0 == 1 else (lambda a, b: (None, None))
    if seed is not None:
        torch.manual_seed(seed)
    s, t, outs = 0, None, []
    for t in opt_ts:
        t = t // window * window
        outs.append(vc_segment(hubert_sd, cpt, audio_pad[s: t + t_pad2 + window], *sl(s // window, (t + t_pad2) // window),
                               index, big_npy, index_rate, version, protect)[t_pad_tgt: -t_pad_tgt])
        s = t
    outs.append(vc_segment(hubert_sd, cpt, audio_pad[t:], *sl(t // window if t is not None else 0, None),
                           index, big_npy, index_rate, version, protect)[t_pad_tgt: -t_pad_tgt])
    audio_opt = np.concatenate(outs)
    float_out = audio_opt.copy()
    if rms_mix_rate != 1:
        audio_opt = change_rms(audio, 16000, audio_opt, tgt_sr, rms_mix_rate)
    audio_max = np.abs(audio_opt).max() / 0.99
    max_int16 = 32768
    if audio_max > 1:
        max_int16 /= audio_max
    mixed = audio_opt.copy()
    out_i16 = (audio_opt * max_int16).astype(np.int16)
    if return_all:
        return out_i16, dict(float_out=float_out, mixed=mixed, pitch=pitch, pitchf=pitchf, opt_ts=opt_ts, f0=f0)
    return out_i16
