"""TEST INFRASTRUCTURE ONLY — CPU restatement of the `mangio-crepe` F0 path of the reference
(`VC.get_f0_crepe_computation`, vc_infer_pipeline.py:96-137, selected at :310-313).

The reference's own lines (quantile normalisation, the `torchcrepe.predict` call with `batch_size = hop_length * 2`,
`pad=True`, the `source < 0.001 -> nan` rule and the `np.interp` resize) are restated from the reference repository.  Everything
inside `torchcrepe.predict` is a THIRD-PARTY dependency absent from the reference repository — `torchcrepe==0.0.20`
(requirements.txt:19) — restated here from its published source (torchcrepe/{core,model,decode,convert}.py and
librosa.sequence.viterbi): PARITY UNPINNED (no torchcrepe, no librosa, no `full.pth` in this environment):

  preprocess : resample to 16 kHz if needed; zero-pad 512 each side; frames of 1024 at `hop_length`; per frame subtract the
               mean and divide by max(1e-10, std) (unbiased std)
  model      : Crepe('full'): 6 x [zero-pad, Conv2d(k x 1), ReLU, BatchNorm2d(eps 0.0010000000474974513), MaxPool (2,1)]
               (1024, 128, 128, 128, 256, 512 channels; kernel 512 stride 4 pad (254,254) first, then kernel 64 pad (31,32)),
               flatten (position-major), Linear(2048, 360), sigmoid
  postprocess: bins outside [fmin, fmax) set to -inf; decoder = viterbi: softmax over bins, librosa.sequence.viterbi with the
               triangular transition max(12 - |i - j|, 0) (row-normalised); bins -> cents = 20 bin + 1997.3794084376191 plus a
               TRIANGULAR RANDOM DITHER of +-20 cents (scipy.stats.triang.rvs — the reference's output is random!) -> Hz
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]
SAMPLE_RATE, WINDOW, PITCH_BINS, CENTS_PER_BIN = 16000, 1024, 360, 20
CENTS_OFFSET = 1997.3794084376191
BN_EPS = 0.0010000000474974513
CHANNELS = [1024, 128, 128, 128, 256, 512]          # torchcrepe model 'full'


def frames_from_audio(audio: np.ndarray, hop: int) -> torch.Tensor:
    """torchcrepe.preprocess (pad=True) for 16 kHz mono input: [n_frames, 1024] normalised frames."""
    a = torch.from_numpy(np.asarray(audio, dtype=np.float32))[None]
    total = 1 + a.shape[1] // hop
    a = F.pad(a, (WINDOW // 2, WINDOW // 2))
    frames = F.unfold(a[:, None, None, :], kernel_size=(1, WINDOW), stride=(1, hop))
    frames = frames.transpose(1, 2).reshape(-1, WINDOW)[:total]
    frames = frames - frames.mean(dim=1, keepdim=True)
    return frames / torch.max(torch.tensor(1e-10), frames.std(dim=1, keepdim=True))


def model(sd: SD, frames: torch.Tensor) -> torch.Tensor:
    """torchcrepe.Crepe.forward: [n, 1024] -> sigmoid activations [n, 360]."""
    with torch.no_grad():
        x = frames[:, None, :, None]
        for i in range(6):
            pad = (0, 0, 254, 254) if i == 0 else (0, 0, 31, 32)
            x = F.pad(x, pad)
            x = F.conv2d(x, sd[f"conv{i + 1}.weight"], sd[f"conv{i + 1}.bias"], stride=(4, 1) if i == 0 else (1, 1))
            x = F.relu(x)
            p = f"conv{i + 1}_BN"
            x = F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False, 0.0, BN_EPS)
            x = F.max_pool2d(x, (2, 1), (2, 1))
        x = x.permute(0, 2, 1, 3).reshape(x.shape[0], -1)
        return torch.sigmoid(F.linear(x, sd["classifier.weight"], sd["classifier.bias"]))


def frequency_to_bins(f: float, ceil: bool = False) -> int:
    b = (1200.0 * np.log2(f / 10.0) - CENTS_OFFSET) / CENTS_PER_BIN
    return int(np.ceil(b) if ceil else np.floor(b))


def transition_matrix() -> np.ndarray:
    xx, yy = np.meshgrid(range(PITCH_BINS), range(PITCH_BINS))
    t = np.maximum(12 - abs(xx - yy), 0).astype(np.float64)
    return t / t.sum(axis=1, keepdims=True)


def viterbi_states(prob: np.ndarray, transition: np.ndarray) -> np.ndarray:
    """librosa.sequence.viterbi(prob [n_states, n_steps], transition): most likely state sequence, uniform initial
    distribution, log domain with `tiny` added before the logs."""
    n_states, n_steps = prob.shape
    tiny = np.finfo(prob.dtype if prob.dtype.kind == "f" else np.float64).tiny
    log_trans = np.log(transition + tiny)
    log_prob = np.log(prob.T + tiny)
    log_p_init = np.log(np.full(n_states, 1.0 / n_states) + tiny)
    value = np.zeros((n_steps, n_states))
    ptr = np.zeros((n_steps, n_states), dtype=np.int64)
    value[0] = log_prob[0] + log_p_init
    for t in range(1, n_steps):
        trans_out = value[t - 1] + log_trans.T            # [to, from]
        ptr[t] = np.argmax(trans_out, axis=1)
        value[t] = log_prob[t] + trans_out[np.arange(n_states), ptr[t]]
    states = np.zeros(n_steps, dtype=np.int64)
    states[-1] = np.argmax(value[-1])
    for t in range(n_steps - 2, -1, -1):
        states[t] = ptr[t + 1, states[t + 1]]
    return states


def decode_viterbi(activ: torch.Tensor, fmin: float, fmax: float) -> np.ndarray:
    """torchcrepe.postprocess + decode.viterbi: sigmoid activations [n, 360] -> bins [n]."""
    p = activ.clone().t()[None]                              # [1, 360, n]
    p[:, :frequency_to_bins(fmin)] = -float("inf")
    p[:, frequency_to_bins(fmax, ceil=True):] = -float("inf")
    probs = torch.softmax(p, dim=1)[0].numpy()               # float32, like probs.cpu().numpy() in torchcrepe
    return viterbi_states(probs, transition_matrix())


def bins_to_frequency(bins: np.ndarray, rng: Optional[np.random.Generator] = None) -> np.ndarray:
    """torchcrepe.convert.bins_to_frequency: cents (+ triangular dither of +-20 cents when `rng` is given; torchcrepe always
    dithers, with scipy's global RNG) -> Hz, float32 like the torch tensors there."""
    cents = (CENTS_PER_BIN * bins + CENTS_OFFSET).astype(np.float32)
    if rng is not None:
        cents = cents + rng.triangular(-CENTS_PER_BIN, 0.0, CENTS_PER_BIN, size=cents.shape).astype(np.float32)
    return (10.0 * 2.0 ** (cents / 1200.0)).astype(np.float32)


def get_f0_crepe_computation(sd: SD, x: np.ndarray, f0_min: float, f0_max: float, p_len: Optional[int], hop_length: int = 160,
                             rng: Optional[np.random.Generator] = None, return_all: bool = False):
    """VC.get_f0_crepe_computation (vc_infer_pipeline.py:96-137) with model='full'."""
    x = x.astype(np.float32)
    x = x / np.quantile(np.abs(x), 0.999)
    frames = frames_from_audio(x, hop_length)
    activ = torch.cat([model(sd, frames[i:i + 2 * hop_length]) for i in range(0, frames.shape[0], 2 * hop_length)])
    bins = decode_viterbi(activ, f0_min, f0_max)
    pitch = bins_to_frequency(bins, rng)
    p_len = p_len or x.shape[0] // hop_length
    source = np.array(pitch, dtype=np.float32)
    source[source < 0.001] = np.nan
    target = np.interp(np.arange(0, len(source) * p_len, len(source)) / p_len, np.arange(0, len(source)), source)
    f0 = np.nan_to_num(target)
    if return_all:
        return f0, dict(activ=activ, bins=bins, pitch=pitch, frames=frames)
    return f0
