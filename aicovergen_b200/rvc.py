"""Host mirror of the reference's src/rvc.py: `Config`, `load_hubert`, `get_vc`, `rvc_infer` with the same
signatures and return values, building GPU operator objects instead of torch modules.

  Config(device, is_half)            rvc.py:20-95   -> same attributes; segmentation constants are outputs-defining
  load_hubert(device, is_half, path) rvc.py:98-109  -> HubertB200 (fairseq checkpoint dict {"model": state_dict} or a bare state dict)
  get_vc(device, is_half, config, p) rvc.py:112-143 -> (cpt, version, net_g, tgt_sr, vc)
  rvc_infer(...16 positional...)     rvc.py:146-151 -> writes the converted wav
"""
from __future__ import annotations

from multiprocessing import cpu_count
from pathlib import Path

import numpy as np
import torch
from scipy.io import wavfile

from .hubert import HubertB200
from .synth import SynthesizerB200
from .vc_infer_pipeline import VC

BASE_DIR = Path(__file__).resolve().parent.parent


class Config:
    def __init__(self, device, is_half):
        self.device = device
        self.is_half = is_half
        self.n_cpu = 0
        self.gpu_name = None
        self.gpu_mem = None
        self.x_pad, self.x_query, self.x_center, self.x_max = self.device_config()

    def device_config(self) -> tuple:
        if not torch.cuda.is_available():
            # the reference silently falls back to CPU here (rvc.py:68-71); this build has no CPU path
            raise RuntimeError("b200vc: no CUDA device available (the GPU hot path has no CPU fallback)")
        i_device = int(str(self.device).split(":")[-1]) if ":" in str(self.device) else 0
        name = torch.cuda.get_device_name(i_device)
        # rvc.py:33-50 forces fp32 on 16xx/10xx/P40 boards (and rewrites training configs, not reproduced)
        if (("16" in name and "V100" not in name.upper()) or "P40" in name.upper() or "1060" in name
                or "1070" in name or "1080" in name):
            self.gpu_name = name
            self.is_half = False
        self.gpu_mem = int(torch.cuda.get_device_properties(i_device).total_memory / 1024 / 1024 / 1024 + 0.4)
        if self.n_cpu == 0:
            self.n_cpu = cpu_count()
        if self.is_half:
            x_pad, x_query, x_center, x_max = 3, 10, 60, 65      # rvc.py:76-81
        else:
            x_pad, x_query, x_center, x_max = 1, 6, 38, 41       # rvc.py:82-87
        if self.gpu_mem is not None and self.gpu_mem <= 4:
            x_pad, x_query, x_center, x_max = 1, 5, 30, 32       # rvc.py:89-93
        return x_pad, x_query, x_center, x_max


def load_hubert(device, is_half, model_path):
    """fairseq `checkpoint_utils.load_model_ensemble_and_task([path])` replacement: the checkpoint's "model"
    state dict is all the GPU encoder needs."""
    ck = model_path if isinstance(model_path, dict) else torch.load(model_path, map_location="cpu", weights_only=False)
    sd = ck["model"] if isinstance(ck, dict) and "model" in ck else ck
    hubert = HubertB200(sd, device)
    return hubert.eval()


def get_vc(device, is_half, config, model_path):
    cpt = model_path if isinstance(model_path, dict) else torch.load(model_path, map_location="cpu", weights_only=False)
    if "config" not in cpt or "weight" not in cpt:
        raise ValueError(f"Incorrect format for {model_path}. Use a voice model trained using RVC v2 instead.")
    tgt_sr = cpt["config"][-1]
    cpt["config"][-3] = cpt["weight"]["emb_g.weight"].shape[0]
    version = cpt.get("version", "v1")
    net_g = SynthesizerB200(cpt, device)
    vc = VC(tgt_sr, config)
    return cpt, version, net_g, tgt_sr, vc


def load_audio(file, sr):
    """Mono float32 at `sr`. The reference shells out to ffmpeg (my_utils.py:5-21); here WAV files are read
    directly and resampled with a polyphase filter (ingest is SURVEY.md §8(f) rank 2)."""
    from math import gcd

    from scipy.signal import resample_poly

    file = str(file).strip(" ").strip('"').strip("\n").strip('"').strip(" ")
    in_sr, data = wavfile.read(file)
    if data.dtype.kind == "i":
        data = data.astype(np.float32) / float(np.iinfo(data.dtype).max + 1)
    elif data.dtype.kind == "u":
        data = (data.astype(np.float32) - 128.0) / 128.0
    data = data.astype(np.float32)
    if data.ndim == 2:
        data = data.mean(axis=1)
    if in_sr != sr:
        g = gcd(int(in_sr), int(sr))
        data = resample_poly(data, sr // g, in_sr // g).astype(np.float32)
    return data.flatten()


def rvc_infer(index_path, index_rate, input_path, output_path, pitch_change, f0_method, cpt, version, net_g,
              filter_radius, tgt_sr, rms_mix_rate, protect, crepe_hop_length, vc, hubert_model):
    audio = load_audio(input_path, 16000)
    times = [0, 0, 0]
    if_f0 = cpt.get("f0", 1)
    audio_opt = vc.pipeline(hubert_model, net_g, 0, audio, input_path, times, pitch_change, f0_method, index_path,
                            index_rate, if_f0, filter_radius, tgt_sr, 0, rms_mix_rate, version, protect, crepe_hop_length)
    wavfile.write(output_path, tgt_sr, audio_opt)
