"""GPU-native RMVPE F0 estimator — drop-in for the reference `RMVPE` object at the plug point
`vc.model_rmvpe.infer_from_audio(x, thred=0.03)` (vc_infer_pipeline.py:322-329; rmvpe.py:328-409).

log-mel front-end as a windowed-DFT GEMM, the DeepUnet as NHWC tap-GEMM convolutions with
BatchNorm folded into the weights, the BiGRU as a cluster kernel, and the cents decode in the
reference's numpy summation order — all through libb200vc.so.  The decoded F0 feeds an argmax /
coarse-pitch quantiser whose indices must match the reference bit for bit (BASELINE.json
north_star), so the U-Net runs on the tensor cores with 3xTF32 split operands (fp32-level accuracy, ~2^-22
relative) rather than plain TF32; the front-end DFT, the GRU projections and the salience head
stay on the exact-fp32 kernel, which is also available for the whole net (backend=BACKEND_SIMT).
"""
from __future__ import annotations

import dataclasses
import math
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _ffi, ops
from . import tapgemm as tg
from .plans import PlanCache, StepGraph
from .tapgemm import Epi

BN_EPS = 1e-5
N_FFT, HOP, N_MELS, N_CLASS = 1024, 160, 128, 360


def hz_to_mel_htk(f):
    return 2595.0 * np.log10(1.0 + np.asarray(f, dtype=np.float64) / 700.0)


def mel_to_hz_htk(m):
    return 700.0 * (10.0 ** (np.asarray(m, dtype=np.float64) / 2595.0) - 1.0)


def mel_basis(sr=16000, n_fft=N_FFT, n_mels=N_MELS, fmin=30.0, fmax=8000.0) -> np.ndarray:
    """librosa.filters.mel(htk=True, norm='slaney') as configured at rmvpe.py:277-284, 343-345."""
    n_bins = 1 + n_fft // 2
    fftfreqs = np.linspace(0, sr / 2.0, n_bins)
    mel_f = mel_to_hz_htk(np.linspace(hz_to_mel_htk(fmin), hz_to_mel_htk(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, n_bins))
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w.astype(np.float32)


def _fold_bn(w: torch.Tensor, sd, p: str, out_dim: int = 0):
    """conv (no bias) followed by eval BatchNorm -> (w', b')."""
    g, b = sd[p + ".weight"].float(), sd[p + ".bias"].float()
    mu, var = sd[p + ".running_mean"].float(), sd[p + ".running_var"].float()
    s = g / torch.sqrt(var + BN_EPS)
    shape = [1] * w.dim()
    shape[out_dim] = -1
    return w.float() * s.reshape(shape), b - mu * s


def split3_weights(wp: torch.Tensor) -> torch.Tensor:
    """[taps, N, K] fp32 -> [taps, N, 3K] = [W_hi | W_hi | W_lo] (hi = RN_tf32(W), lo = RN_tf32(W - hi)): the weight side of the
    3xTF32 scheme; the activation side is stored [hi | lo | hi] by the producing epilogue (b200vc.h `split`)."""
    from .synth import round_tf32
    w = wp.float().contiguous()
    hi = round_tf32(w)
    lo = round_tf32((w - hi).contiguous())
    return torch.cat([hi, hi, lo], dim=-1).contiguous()


class _Sp:
    """3xTF32 split activation: planes hi | lo | hi, each `Ct` channels wide, inside t [1, H, W, 3*Ct]; the handle addresses
    columns [col, col + C) of every plane (sub-handles let two producers fill one concat buffer)."""

    def __init__(self, H, W, Ct, dev, t=None, col=0, C=None):
        self.t = t if t is not None else torch.empty(1, H, W, 3 * Ct, device=dev, dtype=torch.float32)
        self.H, self.W, self.Ct, self.col, self.C = H, W, Ct, col, (Ct if C is None else C)

    def sub(self, col, C):
        return _Sp(self.H, self.W, self.Ct, None, self.t, col, C)

    @property
    def plane0(self):
        return self.t[..., self.col:self.col + self.C]

    @property
    def gemm_in(self):
        assert self.col == 0 and self.C == self.Ct
        return self.t


class RMVPEB200:
    def __init__(self, model, is_half: bool = False, device: str = "cuda:0", backend: int = tg.BACKEND_TC,
                 n_blocks: int = 4, n_enc: int = 5, n_inter: int = 4):
        """`model`: path to rmvpe.pt or an already-loaded state dict (E2E(4,1,(2,2)) names).
        backend = BACKEND_TC (default): the U-Net's convolutions run on the tensor cores as 3xTF32 split-operand GEMMs (fp32-level
        accuracy, see split3_weights); BACKEND_SIMT: everything on the exact-fp32 FMA kernel (cross-check)."""
        sd = torch.load(model, map_location="cpu") if isinstance(model, (str, bytes)) or hasattr(model, "__fspath__") else model
        self.device = torch.device(device)
        self.is_half = is_half          # kept for interface parity; arithmetic is fp32 (or TF32 if backend=TC)
        self.backend = backend
        self.n_blocks, self.n_enc, self.n_inter = n_blocks, n_enc, n_inter
        self._plans = PlanCache()
        self._load(sd)

    def _dev(self, t):
        return t.float().contiguous().to(self.device)

    def _block_weights(self, sd, p: str, key: str):
        W = self.W
        w1, b1 = _fold_bn(sd[p + "conv.0.weight"], sd, p + "conv.1")
        w2, b2 = _fold_bn(sd[p + "conv.3.weight"], sd, p + "conv.4")
        W[key + ".w1"], W[key + ".b1"] = self._dev(tg.pack_conv2d(w1)), self._dev(b1)
        W[key + ".w2"], W[key + ".b2"] = self._dev(tg.pack_conv2d(w2)), self._dev(b2)
        if p + "shortcut.weight" in sd:
            W[key + ".ws"] = self._dev(sd[p + "shortcut.weight"][:, :, 0, 0])
            W[key + ".bs"] = self._dev(sd[p + "shortcut.bias"])
        if self.backend == tg.BACKEND_TC:
            for nm in (".w1", ".w2", ".ws"):
                if key + nm in W and W[key + nm].shape[-1] >= 4:
                    W[key + nm + "s"] = split3_weights(W[key + nm])

    def _load(self, sd):
        self.W = W = {}
        # windowed real-DFT basis: rows [cos(0..512) | -sin(0..512)] * hann(periodic), K = 1024
        n = torch.arange(N_FFT, dtype=torch.float64)
        k = torch.arange(N_FFT // 2 + 1, dtype=torch.float64)
        win = torch.hann_window(N_FFT, periodic=True, dtype=torch.float64)
        ang = 2 * math.pi * k[:, None] * n[None, :] / N_FFT
        basis = torch.cat([torch.cos(ang) * win, -torch.sin(ang) * win], 0)      # [1026, 1024]
        W["dft"] = self._dev(basis)
        mb = torch.zeros(N_MELS, 516)
        mb[:, :513] = torch.from_numpy(mel_basis())
        W["mel"] = self._dev(mb)
        bn = "unet.encoder.bn"
        s = float(sd[bn + ".weight"][0] / torch.sqrt(sd[bn + ".running_var"][0] + BN_EPS))
        self.bn_a, self.bn_b = s, float(sd[bn + ".bias"][0] - sd[bn + ".running_mean"][0] * s)
        for i in range(self.n_enc):
            for b in range(self.n_blocks):
                self._block_weights(sd, f"unet.encoder.layers.{i}.conv.{b}.", f"enc{i}.{b}")
        for i in range(self.n_inter):
            for b in range(self.n_blocks):
                self._block_weights(sd, f"unet.intermediate.layers.{i}.conv.{b}.", f"mid{i}.{b}")
        for i in range(self.n_enc):
            p = f"unet.decoder.layers.{i}."
            wt, bt = _fold_bn(sd[p + "conv1.0.weight"], sd, p + "conv1.1", out_dim=1)
            W[f"dec{i}.up.w"], W[f"dec{i}.up.b"] = self._dev(tg.pack_convt2d(wt)), self._dev(bt)
            if self.backend == tg.BACKEND_TC:
                W[f"dec{i}.up.ws"] = split3_weights(W[f"dec{i}.up.w"])
            for b in range(self.n_blocks):
                self._block_weights(sd, p + f"conv2.{b}.", f"dec{i}.{b}")
        W["cnn.w"], W["cnn.b"] = self._dev(tg.pack_conv2d(sd["cnn.weight"])), self._dev(sd["cnn.bias"])
        W["cnn.w2"] = torch.cat([W["cnn.w"], W["cnn.w"]], dim=-1).contiguous()      # split input: x = hi + lo, exact-fp32 kernel
        # GRU: input features arrive as (w, c) = w*3 + c (NHWC flatten); the reference uses c*128 + w
        Hh = sd["fc.0.gru.weight_hh_l0"].shape[1]
        self.hidden = Hh
        wi = []
        for suf in ("", "_reverse"):
            w = sd[f"fc.0.gru.weight_ih_l0{suf}"].float()                       # [3H, 3*128] (c-major)
            wi.append(w.view(3 * Hh, 3, N_MELS).permute(0, 2, 1).reshape(3 * Hh, 3 * N_MELS))
        W["gru.wih"] = self._dev(torch.cat(wi, 0))                               # [2*3H, 384]
        W["gru.bih"] = self._dev(torch.cat([sd["fc.0.gru.bias_ih_l0"], sd["fc.0.gru.bias_ih_l0_reverse"]]))
        W["gru.whh"] = self._dev(torch.stack([sd["fc.0.gru.weight_hh_l0"], sd["fc.0.gru.weight_hh_l0_reverse"]]))
        W["gru.bhh"] = self._dev(torch.stack([sd["fc.0.gru.bias_hh_l0"], sd["fc.0.gru.bias_hh_l0_reverse"]]))
        W["fc.w"], W["fc.b"] = self._dev(sd["fc.1.weight"]), self._dev(sd["fc.1.bias"])

    # ------------------------------------------------------------------
    def _plan(self, n_samples: int) -> "_RmvpePlan":
        return self._plans.get_or_build(n_samples, lambda: _RmvpePlan(self, n_samples))

    @_ffi.on_device
    @torch.no_grad()
    def salience_from_audio(self, audio: torch.Tensor) -> torch.Tensor:
        """Device tensor [n_frames, 360] (rmvpe.py:370-373)."""
        pl = self._plan(int(audio.numel()))
        pl.run(audio)
        return pl.sal[:pl.n_frames]

    @_ffi.on_device
    @torch.no_grad()
    def mel2hidden(self, mel: torch.Tensor) -> torch.Tensor:
        """Reference signature (rmvpe.py:350-357): log-mel [1,128,n] (or [128,n]) -> salience [1,n,360] (device tensor)."""
        m2 = mel.reshape(N_MELS, -1)
        n = int(m2.shape[1])
        pl = self._plan((n - 1) * HOP)
        pl.run_from_logmel(m2.t().to(self.device).float().contiguous())
        return pl.sal[:n].unsqueeze(0)

    def decode(self, hidden, thred: float = 0.03) -> np.ndarray:
        """Reference signature (rmvpe.py:359-364): salience [n,360] (numpy or tensor) -> f0 [n] float64."""
        with torch.cuda.device(self.device):
            h = torch.as_tensor(hidden).to(self.device).float().contiguous()
            n = int(h.shape[0])
            cents = torch.empty(n, device=self.device, dtype=torch.float64)
            f0d = torch.empty(n, device=self.device, dtype=torch.float64)
            ops.rmvpe_decode(h, f0d, n, thred, cents=cents)
            c = cents.cpu().numpy()
        f0 = 10 * (2 ** (c / 1200))
        f0[f0 == 10] = 0
        return f0

    @_ffi.on_device
    @torch.no_grad()
    def infer_from_audio_device(self, audio: torch.Tensor, thred: float = 0.03) -> torch.Tensor:
        """f0 [n_frames] float64 on the device (no host sync)."""
        pl = self._plan(int(audio.numel()))
        pl.run(audio)
        ops.rmvpe_decode(pl.sal, pl.f0, pl.n_frames, thred)
        return pl.f0

    @_ffi.on_device
    def infer_from_audio_begin(self, audio, thred: float = 0.03):
        """First half of infer_from_audio: enqueue the network, the decode and the D2H of the cents track (into pinned memory)
        on the CURRENT stream and return a handle without waiting — a caller that runs this on a side stream overlaps the F0
        estimate (whose BiGRU occupies 16 SMs for tens of ms) with other work."""
        if isinstance(audio, torch.Tensor):
            a = audio.detach().to(self.device).float().contiguous()      # extension: device tensor in, no H2D
        else:
            a = torch.from_numpy(np.ascontiguousarray(audio)).float().to(self.device)
        pl = self._plan(int(a.numel()))
        pl.run(a)
        ops.rmvpe_decode(pl.sal, pl.f0, pl.n_frames, thred, cents=pl.cents)
        if getattr(pl, "cents_host", None) is None:
            pl.cents_host = torch.empty(pl.cents.shape, dtype=pl.cents.dtype).pin_memory()
        pl.cents_host.copy_(pl.cents, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        return pl, done, a

    def infer_from_audio_end(self, handle) -> np.ndarray:
        pl, done, _ = handle
        done.synchronize()
        cents_pred = pl.cents_host.numpy().copy()
        # the reference's own last two numpy lines (rmvpe.py:361-362), on the host so f0 is bit-identical
        f0 = 10 * (2 ** (cents_pred / 1200))
        f0[f0 == 10] = 0
        return f0

    def infer_from_audio(self, audio: np.ndarray, thred: float = 0.03) -> np.ndarray:
        """Reference signature (rmvpe.py:366-383): np.ndarray[N] -> np.ndarray[1 + N//160] (float64 Hz, 0 = unvoiced)."""
        return self.infer_from_audio_end(self.infer_from_audio_begin(audio, thred))


class _RmvpePlan:
    def __init__(self, m: RMVPEB200, n_samples: int):
        dev, W, be = m.device, m.W, m.backend
        f32 = dict(device=dev, dtype=torch.float32)
        steps: List = []
        add = steps.append
        self.n_samples = n_samples
        nf = 1 + n_samples // HOP
        self.n_frames = nf
        T = 32 * ((nf - 1) // 32 + 1)
        self.T = T
        pad = N_FFT // 2
        self.audio = torch.empty(n_samples, **f32)
        padded = torch.zeros(n_samples + 2 * pad + 8, **f32)
        add(lambda: ops.reflect_pad_1d(self.audio, padded, pad))
        # ---- log-mel: frames (overlapping rows, stride HOP) x windowed DFT basis, magnitude, mel GEMM
        spec = torch.empty(nf, 2 * (N_FFT // 2 + 1), **f32)
        frames = tg.View(padded, (N_FFT, nf, 1, 1, 1), (1, HOP, 0, 0, 0))
        add(tg.TapGemm(frames, tg.weights(W["dft"]), [(0, 0, 0, 0, 0)], (nf, 1, 1), tg.out_of(spec), None, tg.BACKEND_SIMT, name="stft"))
        mag = torch.empty(nf, 516, **f32)
        add(lambda: ops.magnitude(spec, mag, N_FFT // 2 + 1))
        melp = torch.empty(nf, N_MELS, **f32)
        add(tg.linear(mag, W["mel"], melp, None, tg.BACKEND_SIMT, name="mel"))
        img = torch.empty(1, T, N_MELS, 1, **f32)        # NHWC: H = frames, W = mel bins, C = 1
        self.n_front = len(steps)                        # steps before this one build `melp` from audio
        self.melp, self.mel_is_log, self.img = melp, False, img
        add(lambda: ops.logmel_affine_reflect(melp, img.view(T, N_MELS), nf, -1.0 if self.mel_is_log else 1e-5, m.bn_a, m.bn_b))

        S = be == tg.BACKEND_TC          # tensor-core path = 3xTF32 split operands; everything else exact-fp32 SIMT
        ex = tg.BACKEND_SIMT
        # The tensor core rounds its fp32 accumulator toward zero at every K=8 step, so a long reduction (9 taps x 3 x 512
        # channels = 1728 steps) drifts by ~1e-4 relative — too much for bit-exact F0 indices.  Reductions longer than KMAX
        # are therefore split over several launches (subsets of the taps) whose partial sums are added on the CUDA cores
        # (round-to-nearest) through the epilogue's `acc_in`; every accumulation chain stays <= KMAX / 8 steps.
        KMAX = int(__import__("os").environ.get("B200VC_RMVPE_KMAX", "1728"))
        scratch = torch.empty(T * N_MELS * 5 + 65536, **f32) if S else None

        def add_tc(op):
            p = op.params
            if op.backend != tg.BACKEND_TC or p.Kc * p.ntaps <= KMAX:
                return add(op)
            per = max(1, KMAX // p.Kc)
            groups = [op.taps[i:i + per] for i in range(0, len(op.taps), per)]
            space = (p.OW, p.OH, p.OB)
            nel = p.OB * p.OH * p.OW * p.N
            assert nel <= scratch.numel(), (op.name, nel, scratch.numel())
            scr = scratch[:nel].view(p.OB, p.OH, p.OW, p.N)
            for gi, g in enumerate(groups):
                if gi < len(groups) - 1:
                    add(tg.TapGemm(op.a, op.w, g, space, tg.out_of(scr), Epi(acc_in=scr if gi else None), op.backend,
                                   box=(p.BW, p.BH), name=f"{op.name}.k{gi}"))
                else:
                    add(tg.TapGemm(op.a, op.w, g, space, op.out, dataclasses.replace(op.epi, acc_in=scr), op.backend,
                                   box=(p.BW, p.BH), name=op.name))

        def new(H_, W_, C_):
            return _Sp(H_, W_, C_, dev) if S else torch.empty(1, H_, W_, C_, **f32)

        def block(x, key, out, H_, W_, cout):
            """ConvBlockRes (rmvpe.py:23-58).  x / out: _Sp handles on the tensor-core path (x is the plain 1-channel image for
            the very first block), plain NHWC tensors on the SIMT path."""
            t1 = new(H_, W_, cout)
            b1, b2 = W[key + ".b1"], W[key + ".b2"]
            if not S:
                add(tg.conv2d(x, W[key + ".w1"], t1, 3, 3, (1, 1), Epi(bias=b1, act_pre=tg.ACT_RELU), ex, name=key + ".c1"))
                sc = x
                if key + ".ws" in W:
                    sc = torch.empty(1, H_, W_, cout, **f32)
                    add(tg.linear(x, W[key + ".ws"], sc, Epi(bias=W[key + ".bs"]), ex, name=key + ".sc"))
                add(tg.conv2d(t1, W[key + ".w2"], out, 3, 3, (1, 1), Epi(bias=b2, act_pre=tg.ACT_RELU, res=sc), ex, name=key + ".c2"))
                return
            first = not isinstance(x, _Sp)       # Cin = 1: not TMA-addressable, stays on the exact-fp32 kernel
            xin = x if first else x.gemm_in
            add_tc(tg.conv2d(xin, W[key + (".w1" if first else ".w1s")], t1.plane0, 3, 3, (1, 1),
                             Epi(bias=b1, act_pre=tg.ACT_RELU, split_out=t1.Ct), ex if first else be, name=key + ".c1"))
            if key + ".ws" in W:
                sc = torch.empty(1, H_, W_, cout, **f32)
                add_tc(tg.linear(xin, W[key + (".ws" if first else ".wss")], sc, Epi(bias=W[key + ".bs"]), ex if first else be, name=key + ".sc"))
                epi2 = Epi(bias=b2, act_pre=tg.ACT_RELU, res=sc, split_out=out.Ct)
            else:
                epi2 = Epi(bias=b2, act_pre=tg.ACT_RELU, res=x.plane0, res_split=x.Ct, split_out=out.Ct)
            add_tc(tg.conv2d(t1.gemm_in, W[key + ".w2s"], out.plane0, 3, 3, (1, 1), epi2, be, name=key + ".c2"))

        # ---- encoder (rmvpe.py:61-119): level output goes straight into the decoder's concat buffer
        x = img
        H_, W_, cout = T, N_MELS, int(W["enc0.0.w1"].shape[1])
        cats = []
        for i in range(m.n_enc):
            cat = new(H_, W_, 2 * cout)
            cats.append((cat, H_, W_, cout))
            for b in range(m.n_blocks):
                last = b == m.n_blocks - 1
                if last:
                    out = cat.sub(cout, cout) if S else cat[..., cout:]
                else:
                    out = new(H_, W_, cout)
                block(x, f"enc{i}.{b}", out, H_, W_, cout)
                x = out
            pooled = new(H_ // 2, W_ // 2, cout)
            if S:
                add(lambda x=x, pooled=pooled: ops.avgpool2x2_split(x.plane0, x.Ct, pooled.plane0, pooled.Ct))
            else:
                add(lambda x=x, pooled=pooled: ops.avgpool2x2(x, pooled))
            x = pooled
            H_, W_, cout = H_ // 2, W_ // 2, cout * 2
        # ---- intermediate (rmvpe.py:122-138)
        for i in range(m.n_inter):
            for b in range(m.n_blocks):
                out = new(H_, W_, cout)
                block(x, f"mid{i}.{b}", out, H_, W_, cout)
                x = out
        # ---- decoder (rmvpe.py:141-187)
        for i in range(m.n_enc):
            cat, Hc, Wc, cc = cats[-1 - i]
            if S:
                ups = tg.conv_transpose2d_s2(x.gemm_in, W[f"dec{i}.up.ws"], cat.sub(0, cc).plane0, 3, 1,
                                             Epi(bias=W[f"dec{i}.up.b"], act_pre=tg.ACT_RELU, split_out=cat.Ct), be, name=f"dec{i}.up")
            else:
                ups = tg.conv_transpose2d_s2(x, W[f"dec{i}.up.w"], cat[..., :cc], 3, 1,
                                             Epi(bias=W[f"dec{i}.up.b"], act_pre=tg.ACT_RELU), ex, name=f"dec{i}.up")
            for op in ups:
                add_tc(op)
            x = cat
            for b in range(m.n_blocks):
                out = new(Hc, Wc, cc)
                block(x, f"dec{i}.{b}", out, Hc, Wc, cc)
                x = out
        # ---- head (rmvpe.py:241-258): N = 3 output channels -> exact-fp32 kernel; on the split path it reads hi + lo
        feat = torch.empty(1, T, N_MELS, 3, **f32)
        if S:
            add(tg.conv2d(x.t[..., :2 * x.Ct], W["cnn.w2"], feat, 3, 3, (1, 1), Epi(bias=W["cnn.b"]), ex, name="cnn"))
        else:
            add(tg.conv2d(x, W["cnn.w"], feat, 3, 3, (1, 1), Epi(bias=W["cnn.b"]), ex, name="cnn"))
        be = ex                                # GRU input projection and salience head: exact fp32
        self.feat, self.n_unet_end = feat, len(steps)
        Hh = m.hidden
        xp = torch.empty(T, 2 * 3 * Hh, **f32)
        add(tg.linear(feat.view(T, 3 * N_MELS), W["gru.wih"], xp, Epi(bias=W["gru.bih"]), be, name="gru.in"))
        hseq = torch.empty(T, 2 * Hh, **f32)
        add(lambda: ops.bigru(xp, W["gru.whh"], W["gru.bhh"], hseq, Hh))
        self.sal = torch.empty(T, N_CLASS, **f32)
        add(tg.linear(hseq, W["fc.w"], self.sal, Epi(bias=W["fc.b"], act_pre=tg.ACT_SIGMOID), be, name="fc"))
        self.f0 = torch.empty(nf, device=dev, dtype=torch.float64)
        self.cents = torch.empty(nf, device=dev, dtype=torch.float64)
        self.steps = steps
        self.graph = StepGraph(steps)

    def run(self, audio: torch.Tensor):
        self.audio.copy_(audio.reshape(-1))
        self.mel_is_log = False
        self.graph()

    def run_from_logmel(self, mel_t: torch.Tensor):
        """mel_t [n_frames, 128] log-mel (what MelSpectrogram.forward returns, transposed): skips the front-end."""
        self.melp.copy_(mel_t)
        self.mel_is_log = True
        for st in self.steps[self.n_front:]:
            st()
        self.mel_is_log = False
