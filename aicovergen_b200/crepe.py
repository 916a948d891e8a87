"""GPU-native crepe F0 estimator for `f0_method="mangio-crepe"` — stands where `torchcrepe.predict(...)` stands in
`VC.get_f0_crepe_computation` (vc_infer_pipeline.py:96-137; `torchcrepe==0.0.20`, requirements.txt:19, model 'full').

torchcrepe is a third-party dependency that is not in the reference repository; its published algorithm is restated (see
oracle/crepe.py for the line-by-line CPU restatement and the PARITY UNPINNED note):

  frames of 1024 samples @16 kHz every `hop_length`, zero-padded by 512, each mean/std normalised        b200vc_crepe_frames
  6 x [pad, Conv2d(k x 1), ReLU, BatchNorm, MaxPool(2,1)]  (1024,128,128,128,256,512 ch; k = 512 s4, then 64)   tap-GEMMs on the tensor cores
                                                                                     + b200vc_maxpool2_affine (BN after ReLU + pool)
  Linear(2048, 360) + sigmoid                                                          tap-GEMM epilogue
  bins outside [fmin, fmax) -> -inf, softmax, log                                      b200vc_crepe_logprob
  librosa.sequence.viterbi with the triangular +-11-bin transition                      b200vc_viterbi_band (one block, fp64)
  bins -> cents (+ torchcrepe's triangular +-20 cent DITHER, host RNG) -> Hz            host, 2 numpy lines like the reference

Work: ~1.4 GMAC per frame (conv2 alone 1.07): a 4-min song at hop 128 is 30 001 frames = 84 TFLOP — as much tensor work as
the MDX passes — processed in batches of `batch_frames` frames through one cached launch plan.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _ffi, ops
from . import tapgemm as tg
from .plans import StepGraph
from .synth import round_tf32
from .tapgemm import Epi

SAMPLE_RATE, WINDOW, PITCH_BINS, CENTS_PER_BIN = 16000, 1024, 360, 20
CENTS_OFFSET = 1997.3794084376191
BN_EPS = 0.0010000000474974513
CHANNELS = [1024, 128, 128, 128, 256, 512]          # torchcrepe model 'full'
FRAME_PITCH = 1536                                   # 254 + 1024 + 254 = 1532 padded frame, rounded to a 16-byte multiple
BAND = 12                                            # transition[i, j] = max(12 - |i - j|, 0), row-normalised


def frequency_to_bins(f: float, ceil: bool = False) -> int:
    """torchcrepe.convert.frequency_to_bins (floor / ceil)."""
    b = (1200.0 * math.log2(f / 10.0) - CENTS_OFFSET) / CENTS_PER_BIN
    return int(math.ceil(b) if ceil else math.floor(b))


class CrepeB200:
    def __init__(self, state_dict: Dict[str, torch.Tensor], device: str = "cuda:0", backend: int = tg.BACKEND_TC,
                 batch_frames: int = 512):
        """`state_dict`: torchcrepe's `full.pth` (conv{1..6}.weight/bias, conv{1..6}_BN.*, classifier.*)."""
        self.device = torch.device(device)
        self.backend = backend
        self.B = int(batch_frames)
        self._plan: Optional[_CrepePlan] = None
        R = backend == tg.BACKEND_TC
        dev = self.device
        rnd = (lambda t: round_tf32(t.float().contiguous())) if R else (lambda t: t.float().contiguous())
        W = {}
        w1 = state_dict["conv1.weight"].float()[:, 0, :, 0]                       # [1024, 512]
        W["c1.w"], W["c1.b"] = rnd(w1).to(dev), state_dict["conv1.bias"].float().to(dev)
        for i in range(2, 7):
            w = state_dict[f"conv{i}.weight"].float()[:, :, :, 0]                  # [Cout, Cin, 64]
            W[f"c{i}.w"] = rnd(tg.pack_conv1d(w)).to(dev)                          # [64, Cout, Cin]
            W[f"c{i}.b"] = state_dict[f"conv{i}.bias"].float().to(dev)
        for i in range(1, 7):
            p = f"conv{i}_BN"
            s = state_dict[p + ".weight"].float() / torch.sqrt(state_dict[p + ".running_var"].float() + BN_EPS)
            W[f"bn{i}.s"] = s.contiguous().to(dev)
            W[f"bn{i}.t"] = (state_dict[p + ".bias"].float() - state_dict[p + ".running_mean"].float() * s).contiguous().to(dev)
        W["fc.w"], W["fc.b"] = rnd(state_dict["classifier.weight"]).to(dev), state_dict["classifier.bias"].float().to(dev)
        self.W = W
        # log transition band [from][d = to - from + 11] (float64, librosa adds tiny(float32) before the log: the decoder input
        # is a float32 array)
        tiny = float(np.finfo(np.float32).tiny)
        xx, yy = np.meshgrid(range(PITCH_BINS), range(PITCH_BINS))
        t = np.maximum(BAND - abs(xx - yy), 0).astype(np.float64)
        t = t / t.sum(axis=1, keepdims=True)
        band = np.full((PITCH_BINS, 2 * BAND - 1), math.log(tiny))
        for k in range(PITCH_BINS):
            for d in range(-(BAND - 1), BAND):
                if 0 <= k + d < PITCH_BINS:
                    band[k, d + BAND - 1] = math.log(t[k, k + d] + tiny)
        self.log_band = torch.from_numpy(band).to(dev)
        self.log_out = math.log(tiny)
        self.log_init = math.log(1.0 / PITCH_BINS + tiny)

    # ------------------------------------------------------------------
    @_ffi.on_device
    @torch.no_grad()
    def activations(self, audio: torch.Tensor, hop_length: int) -> torch.Tensor:
        """audio [N] float32 on the device (already quantile-normalised) -> sigmoid activations [1 + N // hop, 360]."""
        a = audio.reshape(-1).float().contiguous()
        n_frames = 1 + a.numel() // hop_length
        if self._plan is None:
            self._plan = _CrepePlan(self)
        pl = self._plan
        out = torch.empty(n_frames, PITCH_BINS, device=self.device)
        for f0 in range(0, n_frames, self.B):
            nf = min(self.B, n_frames - f0)
            ops.crepe_frames(a, f0, hop_length, WINDOW, pl.frames, 254, nf, self.backend == tg.BACKEND_TC)
            pl.graph()
            out[f0:f0 + nf].copy_(pl.act[:nf])
        return out

    @_ffi.on_device
    @torch.no_grad()
    def viterbi_bins(self, activ: torch.Tensor, fmin: float, fmax: float) -> torch.Tensor:
        """torchcrepe.postprocess + decode.viterbi: activations [n, 360] -> bins [n] (int32, device)."""
        n = int(activ.shape[0])
        logp = torch.empty(n, PITCH_BINS, device=self.device)
        lo, hi = max(0, frequency_to_bins(fmin)), min(PITCH_BINS, frequency_to_bins(fmax, ceil=True))
        ops.crepe_logprob(activ.contiguous(), logp, lo, hi)
        ptr = torch.empty(n, PITCH_BINS, device=self.device, dtype=torch.int16)
        states = torch.empty(n, device=self.device, dtype=torch.int32)
        ops.viterbi_band(logp, self.log_band, self.log_out, self.log_init, ptr, states, BAND)
        return states

    def predict(self, audio, sample_rate: int, hop_length: int, fmin: float, fmax: float, dither_seed: Optional[int] = None,
                dither: bool = True) -> np.ndarray:
        """torchcrepe.predict(audio, sr, hop, fmin, fmax, 'full', decoder=viterbi, pad=True) -> pitch [n_frames] float32 Hz.
        torchcrepe dithers the bin centres with a triangular +-20 cent noise from scipy's global RNG; here the draw uses
        numpy's Generator(dither_seed) (None = fresh entropy), `dither=False` returns the bin centres."""
        if sample_rate != SAMPLE_RATE:
            raise NotImplementedError("the RVC path calls crepe at 16 kHz (vc_infer_pipeline.py:118)")
        a = audio if isinstance(audio, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(audio, dtype=np.float32))
        a = a.to(self.device)
        bins = self.viterbi_bins(self.activations(a, hop_length), fmin, fmax).cpu().numpy()
        cents = (CENTS_PER_BIN * bins + CENTS_OFFSET).astype(np.float32)
        if dither:
            rng = np.random.default_rng(dither_seed)
            cents = cents + rng.triangular(-CENTS_PER_BIN, 0.0, CENTS_PER_BIN, size=cents.shape).astype(np.float32)
        return (10.0 * 2.0 ** (cents / 1200.0)).astype(np.float32)


class _CrepePlan:
    """Buffers + prepared launches of the six conv layers and the classifier for one batch of B frames."""

    def __init__(self, m: CrepeB200):
        dev, W, be, B = m.device, m.W, m.backend, m.B
        R = be == tg.BACKEND_TC
        f32 = dict(device=dev, dtype=torch.float32)
        steps: List = []
        add = steps.append
        self.frames = torch.zeros(B, FRAME_PITCH, **f32)               # zero pads stay zero; the frame is written at [254, 1278)
        # ---- conv1: 512 taps, stride 4, Cin = 1 -> a GEMM over overlapping 512-sample rows (row pitch 4 floats)
        L = 256
        c = torch.empty(B, L, CHANNELS[0], **f32)
        a = tg.View(self.frames, (512, L, B, 1, 1), (1, 4, FRAME_PITCH, 0, 0))
        o = tg.Out(c, 0, L * CHANNELS[0], CHANNELS[0], B, L)
        add(tg.TapGemm(a, tg.weights(W["c1.w"]), [(0, 0, 0, 0, 0)], (L, B, 1), o, Epi(bias=W["c1.b"], act_pre=tg.ACT_RELU), be,
                       name="crepe.conv1"))
        x = torch.empty(B, L // 2, CHANNELS[0], **f32)
        add(lambda c=c, x=x: ops.maxpool2_affine(c, W["bn1.s"], W["bn1.t"], x, R))
        L //= 2
        for i in range(2, 7):
            co = CHANNELS[i - 1]
            c = torch.empty(B, L, co, **f32)
            add(tg.conv1d(x, W[f"c{i}.w"], c, pad=31, epi=Epi(bias=W[f"c{i}.b"], act_pre=tg.ACT_RELU), backend=be, name=f"crepe.conv{i}"))
            x = torch.empty(B, L // 2, co, **f32)
            add(lambda c=c, x=x, i=i: ops.maxpool2_affine(c, W[f"bn{i}.s"], W[f"bn{i}.t"], x, R))
            L //= 2
        assert L == 4 and x.shape[1] * x.shape[2] == W["fc.w"].shape[1]
        self.act = torch.empty(B, PITCH_BINS, **f32)
        add(tg.linear(x.view(B, -1), W["fc.w"], self.act, Epi(bias=W["fc.b"], act_pre=tg.ACT_SIGMOID), be, name="crepe.fc"))
        self.steps = steps
        self.graph = StepGraph(steps)
