"""Host mirror of the reference orchestrator (src/main.py): `song_cover_pipeline` with the reference's 21-argument
signature, plus `CoverEngine`, the array-level form of the same stage graph that keeps every intermediate stem in
HBM (the reference passes WAV files between stages, main.py:166-203).

Stage graph (main.py:166-190, 193-203, 229-233):
    song --MDX(Voc_FT, denoise)--> vocals, instrumental
    vocals --MDX(KARA_2, denoise)--> backup vocals (main stem), main vocals (inverse stem)
    main vocals --MDX(Reverb_HQ, denoise, exclude_main)--> de-reverbed main vocals (inverse stem)
    de-reverbed vocals --mono 16 kHz--> RVC VC.pipeline --> converted vocals @ tgt_sr
    converted vocals --high-pass, compressor, reverb (main.py:206-226)--> effected vocals (int16, as the WAV holds them)
    effected + backup + instrumental --pydub: gains -4/-6/-7 dB, overlay (main.py:229-233)--> cover (int16 frames)

Out of scope here (SURVEY.md §2 rows 10-14): YouTube download, ffmpeg/sox (`pitch_change_all`) and the mp3 ENCODER behind
pydub's export — the cover is written as 16-bit WAV (the frames pydub hands to its encoder).
"""
from __future__ import annotations

import gc
import hashlib
import json
import os
from typing import Dict, Optional

import numpy as np
import torch
from scipy.io import wavfile

from . import _ffi, ops
from . import effects as fx
from .mdx import MDX, MDXModel, run_mdx, run_mdx_arrays, run_mdx_device, _read_wav_44k, _write_wav_pcm16
from .rvc import Config, get_vc, load_hubert, rvc_infer

BASE_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
mdxnet_models_dir = os.path.join(BASE_DIR, "mdxnet_models")
rvc_models_dir = os.path.join(BASE_DIR, "rvc_models")
output_dir = os.path.join(BASE_DIR, "song_output")

# the three separation models of preprocess_song with their model_data.json parameter sets
# (mdxnet_models/model_data.json: Voc_FT-class :282-288, KARA_2-class :212-218, Reverb_HQ-class :247-253)
MDX_STAGES = (
    dict(name="UVR-MDX-NET-Voc_FT", dim_f=3072, dim_t=256, n_fft=7680, stem="Vocals", compensate=1.021),
    dict(name="UVR_MDXNET_KARA_2", dim_f=2048, dim_t=256, n_fft=5120, stem="Instrumental", compensate=1.035),
    dict(name="Reverb_HQ_By_FoxJoy", dim_f=3072, dim_t=512, n_fft=6144, stem="Other", compensate=1.035),
)


SUPPORTED_F0_METHODS = ("rmvpe", "mangio-crepe")


class CoverEngine:
    """All models of one cover job resident on one GPU; `cover(song)` runs the whole stage graph on device arrays."""

    def __init__(self, mdx_weights, hubert_sd, rmvpe_sd, rvc_cpt, index=None, device="cuda:0", mdx_stages=MDX_STAGES):
        from .hubert import HubertB200
        from .rmvpe import RMVPEB200
        from .synth import SynthesizerB200
        from .vc_infer_pipeline import VC

        self.device = device
        self.stages = mdx_stages
        self.mdx = []
        for st, w in zip(mdx_stages, mdx_weights):
            model = MDXModel(device, st["dim_f"], st["dim_t"], st["n_fft"], stem_name=st["stem"], compensation=st["compensate"])
            self.mdx.append(MDX(w, model, int(str(device).split(":")[-1])))
        self.config = Config(device, True)
        self.hubert = HubertB200(hubert_sd, device)
        self.net_g = SynthesizerB200(rvc_cpt, device)
        self.cpt = rvc_cpt
        self.tgt_sr = rvc_cpt["config"][-1]
        self.vc = VC(self.tgt_sr, self.config)
        self.vc.model_rmvpe = RMVPEB200(rmvpe_sd, device=device)
        self.index_path = index or ""

    @_ffi.on_device
    @torch.no_grad()
    def separate(self, song_dev: torch.Tensor, group=None) -> Dict[str, torch.Tensor]:
        """The three MDX passes of preprocess_song on a device tensor [2,N] float32 @44.1k -> stems (device tensors).
        With a torch.distributed `group` the chunk list of every pass is shared by the group's ranks (strong scaling of ONE
        song: chunk ranges per rank, one all-gather of the stem per pass)."""
        vocals, instrumental = run_mdx_device(self.mdx[0], song_dev, denoise=True, group=group)
        backup, main_vocals = run_mdx_device(self.mdx[1], vocals, denoise=True, group=group)
        _, dereverb = run_mdx_device(self.mdx[2], main_vocals, denoise=True, group=group)
        return dict(vocals=vocals, instrumental=instrumental, backup=backup, main=main_vocals, dereverb=dereverb)

    @_ffi.on_device
    @torch.no_grad()
    def convert(self, vocals_44k: torch.Tensor, pitch_change=0, index_rate=0.5, filter_radius=3, rms_mix_rate=0.25,
                protect=0.33, f0_method="rmvpe", crepe_hop_length=128, return_device=False):
        """load_audio (mono 16 kHz, on device) + VC.pipeline. Returns int16 @ tgt_sr: a host array like the reference, or
        (return_device=True) the same samples as a device tensor, without the D2H."""
        n16 = int(vocals_44k.shape[1] * 16000 // 44100)
        mono = torch.empty(n16, device=self.device)
        ops.resample_sinc_mono(vocals_44k.contiguous(), mono, 44100, 16000)
        times = [0, 0, 0]
        self.vc.return_device = bool(return_device)
        try:
            return self.vc.pipeline(self.hubert, self.net_g, 0, mono, "array", times, pitch_change, f0_method, self.index_path,
                                    index_rate, self.cpt.get("f0", 1), filter_radius, self.tgt_sr, 0, rms_mix_rate,
                                    self.cpt.get("version", "v1"), protect, crepe_hop_length)
        finally:
            self.vc.return_device = False

    def effects(self, ai_vocals_i16, reverb_rm_size=0.15, reverb_wet=0.2, reverb_dry=0.8, reverb_damping=0.7) -> torch.Tensor:
        """add_audio_effects (main.py:206-226) on the int16 utterance at tgt_sr (host array or device tensor): the int16
        samples of `..._mixed.wav`, on the device."""
        a = ai_vocals_i16 if isinstance(ai_vocals_i16, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(ai_vocals_i16))
        return fx.add_audio_effects_device(a.to(self.device), self.tgt_sr, reverb_rm_size, reverb_wet, reverb_dry, reverb_damping)

    def mix(self, ai_vocals_i16, backup: torch.Tensor, instrumental: torch.Tensor, main_gain=0, backup_gain=0,
            inst_gain=0) -> torch.Tensor:
        """combine_audio (main.py:229-233): ai_vocals_i16 = the int16 utterance at tgt_sr (host array or device tensor; exactly
        what the caller passes is mixed); backup / instrumental = float stems [2, n] @44.1k in HBM, quantised to the int16
        frames their WAV files would hold.  Returns the cover's int16 frames [n_out, 2] @44.1k on the device."""
        a = ai_vocals_i16 if isinstance(ai_vocals_i16, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(ai_vocals_i16))
        out, rate = fx.combine_audio_device([(a.to(self.device), self.tgt_sr), (fx.pcm16_from_planar(backup), 44100),
                                             (fx.pcm16_from_planar(instrumental), 44100)], main_gain, backup_gain, inst_gain)
        self.cover_rate = rate          # max(tgt_sr, 44100): pydub mixes at the highest of the operands' rates
        return out

    @_ffi.on_device
    def cover_device(self, song_dev: torch.Tensor, main_gain=0, backup_gain=0, inst_gain=0, group=None, reverb_rm_size=0.15,
                     reverb_wet=0.2, reverb_dry=0.8, reverb_damping=0.7, **convert_kw) -> torch.Tensor:
        """song already in HBM -> the cover's int16 frames [n, 2] in HBM (the converted utterance goes through the effects
        and into the mix as a device tensor).
        `group`: ranks of a torch.distributed group work on the SAME song (every rank must call this with the same song):
        MDX chunks and RVC segments are shared, every rank ends with the full cover."""
        stems = self.separate(song_dev, group)
        self.vc.group = group
        try:
            ai = self.convert(stems["dereverb"], return_device=True, **convert_kw)
        finally:
            self.vc.group = None
        ai = self.effects(ai, reverb_rm_size, reverb_wet, reverb_dry, reverb_damping)
        return self.mix(ai, stems["backup"], stems["instrumental"], main_gain, backup_gain, inst_gain)

    @_ffi.on_device
    def cover(self, song: np.ndarray, out: Optional[torch.Tensor] = None, **kw) -> np.ndarray:
        """Host array [2, N] float32 in, the cover's int16 frames [n, 2] out (H2D of the song and D2H of the cover included).
        `out`: optional host int16 tensor [>= n, 2] to receive the frames (pinned memory makes the D2H a single DMA); the
        returned array is then a view of its first n rows."""
        dev = torch.from_numpy(np.ascontiguousarray(song, dtype=np.float32)).to(self.device, non_blocking=True)
        res = self.cover_device(dev, **kw)
        if out is None:
            return res.cpu().numpy()
        if out.dtype != torch.int16 or out.dim() != 2 or out.shape[1] != res.shape[1] or out.shape[0] < res.shape[0] or out.is_cuda:
            raise ValueError(f"cover: `out` must be a host int16 tensor [>= {res.shape[0]}, {res.shape[1]}]")
        view = out[:res.shape[0]]
        view.copy_(res)
        return view.numpy()


# ---------------------------------------------------------------------------------------------------------------
# file-level mirror of the reference functions
# ---------------------------------------------------------------------------------------------------------------
def raise_exception(error_msg, is_webui):
    raise Exception(error_msg)      # gr.Error in the WebUI build of the reference (main.py:81-85)


def display_progress(message, percent, is_webui, progress=None):
    if is_webui and progress is not None:
        progress(percent, desc=message)
    else:
        print(message)


def get_hash(filepath):
    h = hashlib.blake2b()
    with open(filepath, "rb") as f:
        while chunk := f.read(8192):
            h.update(chunk)
    return h.hexdigest()[:11]


def get_rvc_model(voice_model, is_webui):
    model_dir = os.path.join(rvc_models_dir, voice_model)
    pth = idx = None
    for file in os.listdir(model_dir):
        ext = os.path.splitext(file)[1]
        if ext == ".pth":
            pth = file
        if ext in (".index", ".npz"):
            idx = file
    if pth is None:
        raise_exception(f"No model file exists in {model_dir}.", is_webui)
    return os.path.join(model_dir, pth), os.path.join(model_dir, idx) if idx else ""


def get_audio_paths(song_dir):
    orig = inst = dereverb = backup = None
    for file in os.listdir(song_dir):
        if file.endswith("_Instrumental.wav"):
            inst = os.path.join(song_dir, file)
            orig = inst.replace("_Instrumental", "")
        elif file.endswith("_Vocals_Main_DeReverb.wav"):
            dereverb = os.path.join(song_dir, file)
        elif file.endswith("_Vocals_Backup.wav"):
            backup = os.path.join(song_dir, file)
    return orig, inst, dereverb, backup


def convert_to_stereo(audio_path):
    """main.py:125-135 (ffmpeg -ac 2): mono WAVs are duplicated to two channels."""
    sr, data = wavfile.read(audio_path)
    if data.ndim == 1:
        stereo_path = f"{os.path.splitext(audio_path)[0]}_stereo.wav"
        wavfile.write(stereo_path, sr, np.stack([data, data], 1))
        return stereo_path
    return audio_path


def _mdx_model_path(name):
    for ext in (".onnx", ".pt", ".pth"):
        p = os.path.join(mdxnet_models_dir, name + ext)
        if os.path.exists(p):
            return p
    return os.path.join(mdxnet_models_dir, name + ".onnx")


def preprocess_song(song_input, mdx_model_params, song_id, is_webui, input_type, progress=None):
    if input_type == "yt":
        raise_exception("YouTube download is out of scope for this build (no network stack); pass a local file.", is_webui)
    orig_song_path, keep_orig = song_input, True
    song_output_dir = os.path.join(output_dir, song_id)
    orig_song_path = convert_to_stereo(orig_song_path)
    display_progress("[~] Separating Vocals from Instrumental...", 0.1, is_webui, progress)
    vocals_path, instrumentals_path = run_mdx(mdx_model_params, song_output_dir, _mdx_model_path("UVR-MDX-NET-Voc_FT"),
                                              orig_song_path, denoise=True, keep_orig=keep_orig)
    display_progress("[~] Separating Main Vocals from Backup Vocals...", 0.2, is_webui, progress)
    backup_vocals_path, main_vocals_path = run_mdx(mdx_model_params, song_output_dir, _mdx_model_path("UVR_MDXNET_KARA_2"),
                                                   vocals_path, suffix="Backup", invert_suffix="Main", denoise=True)
    display_progress("[~] Applying DeReverb to Vocals...", 0.3, is_webui, progress)
    _, main_vocals_dereverb_path = run_mdx(mdx_model_params, song_output_dir, _mdx_model_path("Reverb_HQ_By_FoxJoy"),
                                           main_vocals_path, invert_suffix="DeReverb", exclude_main=True, denoise=True)
    return orig_song_path, vocals_path, instrumentals_path, main_vocals_path, backup_vocals_path, main_vocals_dereverb_path


def voice_change(voice_model, vocals_path, output_path, pitch_change, f0_method, index_rate, filter_radius, rms_mix_rate,
                 protect, crepe_hop_length, is_webui):
    rvc_model_path, rvc_index_path = get_rvc_model(voice_model, is_webui)
    device = "cuda:0"
    config = Config(device, True)
    hubert_model = load_hubert(device, config.is_half, os.path.join(rvc_models_dir, "hubert_base.pt"))
    cpt, version, net_g, tgt_sr, vc = get_vc(device, config.is_half, config, rvc_model_path)
    rvc_infer(rvc_index_path, index_rate, vocals_path, output_path, pitch_change, f0_method, cpt, version, net_g,
              filter_radius, tgt_sr, rms_mix_rate, protect, crepe_hop_length, vc, hubert_model)
    del hubert_model, cpt
    gc.collect()


def _read_wav_i16(path):
    sr, data = wavfile.read(path)
    if data.dtype != np.int16:
        raise ValueError(f"{path}: 16-bit PCM expected (every stage of the pipeline writes PCM_16), got {data.dtype}")
    return int(sr), data


def add_audio_effects(audio_path, reverb_rm_size, reverb_wet, reverb_dry, reverb_damping):
    """main.py:206-226: HighpassFilter -> Compressor(ratio 4, threshold -15 dB) -> Reverb on the converted vocal, written next
    to it as `<name>_mixed.wav` (16-bit, same rate and channel count)."""
    output_path = f"{os.path.splitext(audio_path)[0]}_mixed.wav"
    sr, data = _read_wav_i16(audio_path)
    if data.ndim != 1:
        raise NotImplementedError("add_audio_effects: mono input only (the RVC output is mono)")
    out = fx.add_audio_effects_device(torch.from_numpy(data).to("cuda:0"), sr, reverb_rm_size, reverb_wet, reverb_dry, reverb_damping)
    wavfile.write(output_path, sr, out.cpu().numpy())
    return output_path


def combine_audio(audio_paths, output_path, main_gain, backup_gain, inst_gain, output_format):
    """main.py:229-233: pydub gains (-4 / -6 / -7 dB + the user's), overlay of backup vocals and instrumental onto the main
    vocals, export.  The mp3 encoder is out of scope: the frames are always written as 16-bit WAV."""
    srcs = []
    for p in audio_paths:
        sr, data = _read_wav_i16(p)
        srcs.append((torch.from_numpy(data).to("cuda:0"), sr))
    out, rate = fx.combine_audio_device(srcs, main_gain, backup_gain, inst_gain)
    wavfile.write(output_path, rate, out.cpu().numpy())


def song_cover_pipeline(song_input, voice_model, pitch_change, keep_files, is_webui=0, main_gain=0, backup_gain=0,
                        inst_gain=0, index_rate=0.5, filter_radius=3, rms_mix_rate=0.25, f0_method="rmvpe",
                        crepe_hop_length=128, protect=0.33, pitch_change_all=0, reverb_rm_size=0.15, reverb_wet=0.2,
                        reverb_dry=0.8, reverb_damping=0.7, output_format="mp3", progress=None):
    """Same positional contract as main.song_cover_pipeline (main.py:236-240); returns the cover's path."""
    try:
        if not song_input or not voice_model:
            raise_exception("Ensure that the song input field and voice model field is filled.", is_webui)
        # options this build does not implement are refused BEFORE any separation / conversion work is done
        if str(song_input).startswith("https://") or str(song_input).startswith("http://"):
            raise_exception("YouTube input is out of scope for this build; pass a local file.", is_webui)
        if pitch_change_all != 0:
            raise_exception("pitch_change_all needs sox (out of scope for this build).", is_webui)
        if f0_method not in SUPPORTED_F0_METHODS:
            raise_exception(f"f0_method {f0_method!r}: this build runs {SUPPORTED_F0_METHODS}.", is_webui)
        display_progress("[~] Starting AI Cover Generation Pipeline...", 0, is_webui, progress)
        with open(os.path.join(mdxnet_models_dir, "model_data.json")) as infile:
            mdx_model_params = json.load(infile)
        input_type = "local"
        song_input = song_input.strip('"')
        if not os.path.exists(song_input):
            raise_exception(f"{song_input} does not exist.", is_webui)
        song_id = get_hash(song_input)
        song_dir = os.path.join(output_dir, song_id)
        if not os.path.exists(song_dir):
            os.makedirs(song_dir)
            (orig_song_path, vocals_path, instrumentals_path, main_vocals_path, backup_vocals_path,
             main_vocals_dereverb_path) = preprocess_song(song_input, mdx_model_params, song_id, is_webui, input_type, progress)
        else:
            vocals_path, main_vocals_path = None, None
            paths = get_audio_paths(song_dir)
            if any(p is None for p in paths) or keep_files:
                (orig_song_path, vocals_path, instrumentals_path, main_vocals_path, backup_vocals_path,
                 main_vocals_dereverb_path) = preprocess_song(song_input, mdx_model_params, song_id, is_webui, input_type, progress)
            else:
                orig_song_path, instrumentals_path, main_vocals_dereverb_path, backup_vocals_path = paths
        pitch_change = pitch_change * 12 + pitch_change_all
        stem = os.path.splitext(os.path.basename(orig_song_path))[0]
        ai_vocals_path = os.path.join(song_dir, f"{stem}_{voice_model}_p{pitch_change}_i{index_rate}_fr{filter_radius}_rms{rms_mix_rate}_pro{protect}_{f0_method}{'' if f0_method != 'mangio-crepe' else f'_{crepe_hop_length}'}.wav")
        if output_format != "wav":
            display_progress("[!] mp3 export needs ffmpeg; writing WAV instead.", 0.0, is_webui, progress)
        ai_cover_path = os.path.join(song_dir, f"{stem} ({voice_model} Ver).wav")
        if not os.path.exists(ai_vocals_path):
            display_progress("[~] Converting voice using RVC...", 0.5, is_webui, progress)
            voice_change(voice_model, main_vocals_dereverb_path, ai_vocals_path, pitch_change, f0_method, index_rate,
                         filter_radius, rms_mix_rate, protect, crepe_hop_length, is_webui)
        display_progress("[~] Applying audio effects to Vocals...", 0.8, is_webui, progress)
        ai_vocals_mixed_path = add_audio_effects(ai_vocals_path, reverb_rm_size, reverb_wet, reverb_dry, reverb_damping)
        display_progress("[~] Combining AI Vocals and Instrumentals...", 0.9, is_webui, progress)
        combine_audio([ai_vocals_mixed_path, backup_vocals_path, instrumentals_path], ai_cover_path, main_gain, backup_gain,
                      inst_gain, output_format)
        if not keep_files:
            for file in (vocals_path, main_vocals_path, ai_vocals_mixed_path):
                if file and os.path.exists(file):
                    os.remove(file)
        return ai_cover_path
    except Exception as e:
        raise_exception(str(e), is_webui)
