"""Vocal effects and the final mix of the cover on the device — stands where `main.add_audio_effects` (pedalboard:
HighpassFilter -> Compressor(ratio 4, threshold -15 dB) -> Reverb; main.py:206-226) and `main.combine_audio` (pydub: gain,
overlay, export; main.py:229-233) stand.  Kernels: csrc/effects.cu (how each recursion is made parallel is written there).

pedalboard 0.7.7 / JUCE and pydub 0.25.1 are third-party dependencies that are not in the reference repository; what they compute is
restated in oracle/effects.c and oracle/mixdown.py (the latter runs CPython's own `audioop`, so the mix arithmetic is pinned).
The constants below are computed in float32 the way the JUCE classes compute them."""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import _ffi

_P, _i64, _i32, _f32 = C.c_void_p, C.c_int64, C.c_int, C.c_float

COMB_TUNINGS = (1116, 1188, 1277, 1356, 1422, 1491, 1557, 1617)        # juce::Reverb, at 44.1 kHz
ALLPASS_TUNINGS = (556, 441, 341, 225)
ALLPASS_TERMS = 32                                                      # 0.5 ** 32 ~ 2e-10 of full scale


class MixSource(C.Structure):
    """b200vc_mix_source (include/b200vc.h)."""
    _fields_ = [("x", C.c_void_p), ("n", C.c_int64), ("used", C.c_int64), ("channels", C.c_int32), ("in_rate", C.c_int32),
                ("out_rate", C.c_int32), ("pad_", C.c_int32), ("gain1", C.c_double), ("gain2", C.c_double)]


_ffi.declare("b200vc_fx_hpf_comp", [_P, _P, _P, _i64, _i32, _i32, _f32, _f32, _f32, _f32, _f32, _f32, _f32, _f32, _P])
_ffi.declare("b200vc_fx_reverb_combs", [_P, _P, _P, _i64, C.POINTER(C.c_int), _f32, _f32, _f32, _i32, _P])
_ffi.declare("b200vc_fx_allpass", [_P, _P, _i64, _i32, _i32, _P])
_ffi.declare("b200vc_fx_finish", [_P, _P, _P, _P, _i64, _f32, _f32, _P])
_ffi.declare("b200vc_pcm16_from_planar", [_P, _i64, _i32, _P, _P])
_ffi.declare("b200vc_pydub_mix", [C.POINTER(MixSource), _P, _i64, _i32, _P])


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@dataclass(frozen=True)
class EffectConstants:
    b0: float
    b1: float
    a1: float
    cte_at: float
    cte_rl: float
    thr: float
    thr_inv: float
    expo: float
    comb_delays: Tuple[int, ...]
    allpass_delays: Tuple[int, ...]
    gain: float
    damp: float
    feedback: float
    wet1: float
    dry: float
    comb_terms: int
    warm: int


def effect_constants(sample_rate: int, room_size: float, wet_level: float, dry_level: float, damping: float, cutoff_hz: float = 50.0,
                     threshold_db: float = -15.0, ratio: float = 4.0, attack_ms: float = 1.0, release_ms: float = 100.0,
                     width: float = 1.0) -> EffectConstants:
    """float32 constants of the three JUCE processors (see oracle/effects.c for the formulas and their sources)."""
    f = np.float32
    sr = int(sample_rate)
    n = np.tan(f(np.pi) * f(cutoff_hz) / f(sr), dtype=f)
    a0inv = f(1.0) / (n + f(1.0))
    b0, b1, a1 = f(1.0) * a0inv, f(-1.0) * a0inv, (n - f(1.0)) * a0inv
    exp_factor = f(-2.0 * math.pi * 1000.0 / float(sr))
    cte = lambda ms: f(0.0) if ms < 1.0e-3 else np.exp(exp_factor / f(ms), dtype=f)
    cte_at, cte_rl = cte(attack_ms), cte(release_ms)
    thr = np.power(f(10.0), f(threshold_db) * f(0.05), dtype=f) if threshold_db > -200.0 else f(0.0)
    thr_inv, expo = f(1.0) / thr, f(1.0) / f(ratio) - f(1.0)
    damp, feedback = f(damping) * f(0.4), f(room_size) * f(0.28) + f(0.7)
    wet, dry = f(wet_level) * f(3.0), f(dry_level) * f(2.0)
    wet1 = f(0.5) * wet * (f(1.0) + f(width))
    # state of the high-pass decays like |a1|^k, of the envelope follower like max(cteAT, cteRL)^k, of the comb damping
    # low-pass like damp^k: lengths after which the discarded part is below float32 resolution
    decay = max(abs(float(a1)), float(cte_at), float(cte_rl))
    warm = 0 if decay <= 0.0 else int(math.ceil(math.log(1.0e-10) / math.log(decay))) if decay < 1.0 else 1 << 62
    warm = min(((warm + 1023) // 1024) * 1024, 1 << 30)
    d = float(damp)
    comb_terms = 1 if d <= 0.0 else max(4, min(256, int(math.ceil(-30.0 * math.log(2.0) / math.log(d))))) if d < 1.0 else 256
    return EffectConstants(float(b0), float(b1), float(a1), float(cte_at), float(cte_rl), float(thr), float(thr_inv), float(expo),
                           tuple((sr * t) // 44100 for t in COMB_TUNINGS), tuple((sr * t) // 44100 for t in ALLPASS_TUNINGS),
                           0.015, float(damp), float(feedback), float(wet1), float(dry), comb_terms, warm)


@torch.no_grad()
def add_audio_effects_device(x_i16: torch.Tensor, sample_rate: int, reverb_rm_size: float, reverb_wet: float, reverb_dry: float,
                             reverb_damping: float, return_float: bool = False):
    """x_i16: the mono int16 samples of the converted vocal (device) -> the int16 samples `add_audio_effects` writes
    (and, with return_float, the float samples before the 16-bit conversion)."""
    if x_i16.dim() != 1 or x_i16.dtype != torch.int16:
        raise NotImplementedError("add_audio_effects: mono int16 input (the RVC output) only")
    x = x_i16.contiguous()
    if x.data_ptr() % 16:
        x = x.clone()                    # a view into a larger buffer: the kernel walks 128-bit groups
    n, dev = x.numel(), x.device
    if n == 0:
        return (x.clone(), torch.empty(0, device=dev)) if return_float else x.clone()
    k = effect_constants(sample_rate, reverb_rm_size, reverb_wet, reverb_dry, reverb_damping)
    if min(k.comb_delays) < 1 or min(k.allpass_delays) < 1:
        raise ValueError(f"add_audio_effects: sample rate {sample_rate} is too low for the reverb's delay lines")
    with torch.cuda.device(dev):           # launches go to the current device's stream
        return _effects_on_current_device(x, n, k, return_float)


def _effects_on_current_device(x, n, k, return_float):
    dev = x.device
    lib, s = _ffi.lib(), _stream()
    comp = torch.empty(n, device=dev)
    a, b = torch.empty(n, device=dev), torch.empty(n, device=dev)
    warm = min(k.warm, ((n + 7) // 8) * 8)               # both multiples of 8: the kernel walks 8-sample groups
    chunk = max(2048, (warm // 4 + 7) // 8 * 8)          # one thread per chunk, each walks warm + chunk samples
    _ffi.check(lib.b200vc_fx_hpf_comp(x.data_ptr(), comp.data_ptr(), b.data_ptr(), n, chunk, warm, k.b0, k.b1, k.a1, k.cte_at, k.cte_rl, k.thr,
                                      k.thr_inv, k.expo, s), "fx_hpf_comp")
    lines = torch.empty(8, n, device=dev)
    delays = (C.c_int * 8)(*k.comb_delays)
    _ffi.check(lib.b200vc_fx_reverb_combs(comp.data_ptr(), lines.data_ptr(), a.data_ptr(), n, delays, k.gain, k.damp, k.feedback,
                                          k.comb_terms, s), "fx_reverb_combs")
    for d in k.allpass_delays:
        _ffi.check(lib.b200vc_fx_allpass(a.data_ptr(), b.data_ptr(), n, d, ALLPASS_TERMS, s), "fx_allpass")
        a, b = b, a
    out = torch.empty(n, device=dev, dtype=torch.int16)
    outf = torch.empty(n, device=dev) if return_float else None
    _ffi.check(lib.b200vc_fx_finish(a.data_ptr(), comp.data_ptr(), out.data_ptr(), None if outf is None else outf.data_ptr(), n,
                                    k.wet1, k.dry, s), "fx_finish")
    return (out, outf) if return_float else out


# ---------------------------------------------------------------------------------------------------------------
# pydub mix
# ---------------------------------------------------------------------------------------------------------------
def db_to_float(db: float) -> float:
    """pydub.utils.db_to_float (amplitude)."""
    return 10 ** (float(db) / 20)


def ratecv_frames(n: int, in_rate: int, out_rate: int) -> int:
    """Number of frames audioop.ratecv(state=None) returns for n input frames."""
    if in_rate == out_rate or n == 0:
        return n
    g = math.gcd(in_rate, out_rate)
    return ((n - 1) * (out_rate // g)) // (in_rate // g) + 1


def ms_slice_frames(n: int, rate: int) -> int:
    """Frames of `seg[0:]` for a pydub segment of n frames: the slice runs over whole milliseconds
    (len(seg) = round(1000 n / rate); int(len * rate / 1000) frames, silence-filled when that is more than n)."""
    ms = round(1000 * (float(n) / rate))
    return int(ms * (rate / 1000.0))


def mix_geometry(frames: Sequence[int], rates: Sequence[int]) -> Tuple[int, List[int], int]:
    """main.overlay(backup).overlay(inst): (frame rate of the result, frames of each rate-converted operand that take part,
    frames of the result)."""
    r1 = max(rates[0], rates[1])
    n1, n2 = ratecv_frames(frames[0], rates[0], r1), ratecv_frames(frames[1], rates[1], r1)
    l1 = ms_slice_frames(n1, r1)
    ov1 = min(n2, l1)
    r2 = max(r1, rates[2])
    if r2 != r1:
        raise NotImplementedError("combine_audio: an instrumental at a higher rate than both vocals would resample the first "
                                  "overlay's result; the pipeline's stems share one rate (44.1 kHz)")
    n3 = ratecv_frames(frames[2], rates[2], r2)
    l2 = ms_slice_frames(l1, r2)
    ov2 = min(n3, l2)
    return r2, [min(n1, l1, l2), min(ov1, l2), ov2], l2


@torch.no_grad()
def pcm16_from_planar(x: torch.Tensor) -> torch.Tensor:
    """A stem [channels, n] float32 on the device -> the int16 frames [n, channels] its PCM_16 WAV file holds."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2
    x = x.contiguous()
    out = torch.empty(x.shape[1], x.shape[0], device=x.device, dtype=torch.int16)
    if x.shape[1]:
        with torch.cuda.device(x.device):
            _ffi.check(_ffi.lib().b200vc_pcm16_from_planar(x.data_ptr(), x.shape[1], x.shape[0], out.data_ptr(), _stream()), "pcm16")
    return out


@torch.no_grad()
def combine_audio_device(sources: Sequence[Tuple[torch.Tensor, int]], main_gain: float = 0, backup_gain: float = 0,
                         inst_gain: float = 0) -> Tuple[torch.Tensor, int]:
    """sources: (int16 samples [n] or [n, channels] on the device, frame rate) of main vocals, backup vocals, instrumental —
    what AudioSegment.from_wav holds.  Returns the int16 frames [n_out, channels] that `export` encodes, and their rate."""
    xs = []
    for x, _ in sources:
        if x.dtype != torch.int16 or x.dim() not in (1, 2):
            raise ValueError("combine_audio: int16 [n] or [n, channels] samples expected")
        xs.append(x.contiguous())
    frames = [int(x.shape[0]) for x in xs]
    chans = [1 if x.dim() == 1 else int(x.shape[1]) for x in xs]
    rates = [int(r) for _, r in sources]
    if min(frames) == 0:
        raise ValueError("combine_audio: empty input")
    rate, used, n_out = mix_geometry(frames, rates)
    channels = max(chans)
    out = torch.empty(n_out, channels, device=xs[0].device, dtype=torch.int16)
    if n_out == 0:
        return out, rate
    gains = ((-4, main_gain), (-6, backup_gain), (-7, inst_gain))
    src = (MixSource * 3)()
    for i in range(3):
        src[i] = MixSource(xs[i].data_ptr(), frames[i], used[i], chans[i], rates[i], rate, 0, db_to_float(gains[i][0]),
                           db_to_float(gains[i][1]))
    if any(x.device != xs[0].device for x in xs):
        raise ValueError("combine_audio: the three operands must live on one device")
    with torch.cuda.device(xs[0].device):
        _ffi.check(_ffi.lib().b200vc_pydub_mix(src, out.data_ptr(), n_out, channels, _stream()), "pydub_mix")
    return out, rate
