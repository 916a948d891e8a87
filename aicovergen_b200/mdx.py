"""GPU-native MDX-Net separation pass — host mirror of the reference's src/mdx.py (`MDXModel`, `MDX`,
`run_mdx`, same signatures) over libb200vc.so.

What changes versus the reference is where the work happens: the reference loops chunk by chunk with four
PCIe crossings per chunk (STFT on GPU -> numpy -> onnxruntime -> torch -> iSTFT -> numpy, mdx.py:187-197).
Here the song is uploaded once, chunks are gathered in batches straight from HBM (pad_wave zeros + STFT
reflect padding fused), the STFT / iSTFT are windowed-DFT tap-GEMMs restricted to the dim_f kept bins, the
TFC-TDF U-Net runs as NHWC tap-GEMMs on the tensor cores with BatchNorm folded, and the iSTFT tail scatters the
trimmed chunk directly into the song-level output (trim / concat / [:-pad] / margin logic of mdx.py:195-197,
107-117 folded into its addressing).  One D2H at the end.

The network itself ("ConvTDFNet") ships inside `.onnx` files that are not in the reference repo; the graph is
restated from the public UVR/KUIELab architecture (SURVEY.md §8(c)) and loaded from a state dict.
"""
from __future__ import annotations

import gc
import hashlib
import math
import os
from typing import Dict, List, Optional

import numpy as np
import torch
from scipy.io import wavfile

from . import _ffi, ops
from . import tapgemm as tg
from .plans import StepGraph
from .synth import round_tf32
from .tapgemm import Epi

stem_naming = {"Vocals": "Instrumental", "Other": "Instruments", "Instrumental": "Vocals", "Drums": "Drumless",
               "Bass": "Bassless"}
BN_EPS = 1e-5


class MDXModel:
    """Geometry of one MDX-Net model (mdx.py:19-35) plus API-compatible stft / istft on device tensors."""

    def __init__(self, device, dim_f, dim_t, n_fft, hop=1024, stem_name=None, compensation=1.000):
        if n_fft <= hop:
            # a periodic Hann window of n_fft <= hop has zeros in its overlap-add envelope: the reference's torch.istft
            # (mdx.py:52-62) raises "window overlap add min: 1" there; refuse up front instead of dividing by zero
            raise RuntimeError(f"MDXModel: n_fft {n_fft} with hop {hop}: window overlap-add envelope has zeros (torch.istft refuses it)")
        self.dim_f, self.dim_t, self.dim_c = dim_f, dim_t, 4
        self.n_fft, self.hop = n_fft, hop
        self.stem_name, self.compensation = stem_name, compensation
        self.n_bins = n_fft // 2 + 1
        self.chunk_size = hop * (dim_t - 1)
        self.device = torch.device(device)
        self._dft = {}

    # ---- windowed DFT bases restricted to the kept bins (built once, fp64 -> fp32 [-> TF32 RN])
    def dft(self, rnd: bool):
        if rnd not in self._dft:
            N, F = self.n_fft, self.dim_f
            n = torch.arange(N, dtype=torch.int64)
            f = torch.arange(F, dtype=torch.int64)
            ang = (2 * math.pi / N) * ((f[:, None] * n[None, :]) % N).double()        # exact argument reduction
            win = torch.hann_window(N, periodic=True, dtype=torch.float64)
            cosw, sinw = torch.cos(ang) * win, torch.sin(ang) * win
            fwd = torch.stack([cosw, -sinw], 1).reshape(2 * F, N)                       # row (f, ri)
            coef = torch.full((F,), 2.0, dtype=torch.float64)
            coef[0] = 1.0
            inv = torch.stack([cosw * coef[:, None], -sinw * coef[:, None]], 1).reshape(2 * F, N).t() / N   # [N, (f,ri)]
            T, chunk = self.dim_t, self.chunk_size
            env = torch.zeros(chunk + N, dtype=torch.float64)
            w2 = win * win
            for t in range(T):
                env[t * self.hop: t * self.hop + N] += w2
            conv = (lambda x: round_tf32(x.float().contiguous())) if rnd else (lambda x: x.float().contiguous())
            self._dft[rnd] = (conv(fwd).to(self.device), conv(inv).to(self.device), env.float().to(self.device))
        return self._dft[rnd]

    @_ffi.on_device
    def stft(self, x: torch.Tensor) -> torch.Tensor:
        """[B,2,chunk] -> [B,4,dim_f,dim_t] (L.re, L.im, R.re, R.im) like mdx.py:37-43 (API path, not the hot path)."""
        B = x.reshape(-1, 2, self.chunk_size).shape[0]
        fwd, _, _ = self.dft(False)
        half = self.n_fft // 2
        padded = torch.empty(B, 2, self.chunk_size + self.n_fft, device=self.device)
        xs = x.reshape(B * 2, self.chunk_size).float().contiguous()
        for i in range(B * 2):
            ops.reflect_pad_1d(xs[i], padded.view(B * 2, -1)[i], half)
        spec2 = torch.empty(B, 2, self.dim_t, 2 * self.dim_f, device=self.device)
        _stft_gemm(padded, fwd, spec2, self, tg.BACKEND_SIMT)()
        s = spec2.view(B, 2, self.dim_t, self.dim_f, 2).permute(0, 1, 4, 3, 2)       # [B, ch, ri, F, T]
        return s.reshape(B, 4, self.dim_f, self.dim_t).contiguous()

    @_ffi.on_device
    def istft(self, x: torch.Tensor, freq_pad=None) -> torch.Tensor:
        """[B,4,dim_f,dim_t] -> [B,2,chunk] like mdx.py:45-54 (API path)."""
        B = x.shape[0]
        _, inv, env = self.dft(False)
        spec2 = x.view(B, 2, 2, self.dim_f, self.dim_t).permute(0, 1, 4, 3, 2).contiguous().view(B, 2, self.dim_t, 2 * self.dim_f)
        frames = torch.empty(B, 2, self.dim_t, self.n_fft, device=self.device)
        tg.linear(spec2.view(-1, 2 * self.dim_f), inv, frames.view(-1, self.n_fft), None, tg.BACKEND_SIMT)()
        out = torch.zeros(2, B * self.chunk_size, device=self.device)
        idx = torch.arange(B, device=self.device, dtype=torch.int64) * self.chunk_size
        ops.mdx_ola_store(frames, env, idx, idx, idx + self.chunk_size, out, self.dim_t, self.n_fft, self.hop,
                          self.chunk_size, 0, 1.0, False)
        return out.view(2, B, self.chunk_size).permute(1, 0, 2).contiguous()


def _stft_gemm(padded, fwd, spec2, model: MDXModel, backend):
    """spec2[b,ch,t,(f,ri)] = sum_n padded[b,ch,t*hop+n] * fwd[(f,ri),n] — frames are overlapping strided rows."""
    B = padded.shape[0]
    plen = padded.shape[2]
    a = tg.View(padded, (model.n_fft, model.dim_t, 2, B, 1), (1, model.hop, plen, 2 * plen, 0))
    T, NF = model.dim_t, 2 * model.dim_f
    o = tg.Out(spec2, 2 * T * NF, T * NF, NF, 2, T)
    return tg.TapGemm(a, tg.weights(fwd), [(0, 0, 0, 0, 0)], (T, 2, B), o, None, backend, name="mdx.stft")


# fp16 storage of the U-Net's activations and GEMM weights (wgmma f16, fp32 accumulate): the same 10-bit mantissa
# as the TF32 path at half the shared-memory / L2 / HBM bytes per FLOP.  Only tensors that live inside the network's launch
# plan change type; the spectrograms on either side stay fp32.
MDX_FP16 = os.environ.get("B200VC_MDX_FP16", "1") == "1"      # default ON (validated r02: 5.5e-4 rel. on the full-size net, F0 / stems
                                                                # within the parity bars); B200VC_MDX_FP16=0 -> fp32 storage, TF32 MMAs


class ConvTDFNetB200:
    """The TFC-TDF U-Net on device: stands where `ort.InferenceSession` stands in the reference (mdx.py:74-77)."""

    def __init__(self, sd: Dict[str, torch.Tensor], device, backend=tg.BACKEND_TC):
        self.device = torch.device(device)
        self.backend = backend
        meta = [int(v) for v in sd["_meta"]]
        (self.dim_f, self.dim_t, self.g, self.l, self.n, self.bn, self.k, self.dim_c) = meta
        # fp16 storage needs every GEMM of the plan on the TMA/wgmma kernels (there is no fp16 SIMT path); the narrowest
        # one is the bottleneck TDF with K = dim_f / 2^n / bn (an fp32-operand fallback GEMM when that is not a multiple of 8,
        # which itself needs K % 4 == 0).  Real UVR geometries (dim_f >= 2048) satisfy it; toy geometries fall back to fp32.
        tdf_k = [(self.dim_f >> lvl) // self.bn for lvl in range(self.n + 1)]
        self.half = bool(MDX_FP16 and backend == tg.BACKEND_TC and all(k_ % 4 == 0 for k_ in tdf_k))
        self.W: Dict[str, torch.Tensor] = {}
        self._plans: Dict[int, "_NetPlan"] = {}
        self._load(sd)

    def _dev(self, t, rnd=True):
        t = t.float().contiguous()
        if rnd and self.half:
            return t.half().to(self.device)          # GEMM weight in fp16 mode
        if rnd and self.backend == tg.BACKEND_TC:
            t = round_tf32(t)
        return t.to(self.device)

    @staticmethod
    def _bn(sd, p):
        s = sd[p + ".weight"].float() / torch.sqrt(sd[p + ".running_var"].float() + BN_EPS)
        return s, sd[p + ".bias"].float() - sd[p + ".running_mean"].float() * s

    def _conv_bn(self, sd, conv, bn, key, pack, out_dim=0):
        s, b = self._bn(sd, bn)
        w = sd[conv + ".weight"].float()
        shape = [1] * w.dim()
        shape[out_dim] = -1
        self.W[key + ".w"] = self._dev(pack(w * s.reshape(shape)))
        self.W[key + ".b"] = self._dev(sd[conv + ".bias"].float() * s + b, False)

    def _tfc_tdf(self, sd, p, key):
        for j in range(self.l):
            self._conv_bn(sd, f"{p}.tfc.H.{j}.0", f"{p}.tfc.H.{j}.1", f"{key}.c{j}", tg.pack_conv2d)
        s1, b1 = self._bn(sd, f"{p}.tdf.1")
        s2, b2 = self._bn(sd, f"{p}.tdf.4")
        W = self.W
        w1, w2 = sd[f"{p}.tdf.0.weight"], sd[f"{p}.tdf.3.weight"]
        W[key + ".w1"] = self._dev(w1)
        # fp16 mode: the second TDF GEMM reads K = F/bn elements per row; TMA needs 16-byte row pitches, so when F/bn is not
        # a multiple of 8 (the bottleneck block: 12) that one GEMM keeps fp32/TF32 operands (its input h is then fp32 too)
        if self.half and w2.shape[1] % 8 != 0:
            W[key + ".w2"] = round_tf32(w2.float().contiguous()).to(self.device)
        else:
            W[key + ".w2"] = self._dev(w2)
        W[key + ".s1"], W[key + ".b1"] = self._dev(s1, False), self._dev(b1, False)
        W[key + ".s2"], W[key + ".b2"] = self._dev(s2, False), self._dev(b2, False)

    def _load(self, sd):
        s, b = self._bn(sd, "first_conv.1")
        w = sd["first_conv.0.weight"].float()[:, :, 0, 0] * s[:, None]                 # [g, 4] -> taps per channel pair
        self.W["first.w4"] = self._dev(w, False)                                        # [g, (ch0re, ch0im, ch1re, ch1im)]
        self.W["first.b"] = self._dev(sd["first_conv.0.bias"].float() * s + b, False)
        for i in range(self.n):
            self._tfc_tdf(sd, f"encoding_blocks.{i}", f"enc{i}")
            self._conv_bn(sd, f"ds.{i}.0", f"ds.{i}.1", f"ds{i}", tg.pack_conv2d)
        self._tfc_tdf(sd, "bottleneck_block", "mid")
        for i in range(self.n):
            self._conv_bn(sd, f"us.{i}.0", f"us.{i}.1", f"us{i}", tg.pack_convt2d, out_dim=1)
            self._tfc_tdf(sd, f"decoding_blocks.{i}", f"dec{i}")
        self.W["final.w"] = self._dev(sd["final_conv.0.weight"].float()[:, :, 0, 0], False)   # [4, c] (row kernel: fp32)
        self.W["final.b"] = self._dev(sd["final_conv.0.bias"], False)

    def plan(self, B: int) -> "_NetPlan":
        pl = self._plans.get(B)
        if pl is None:
            # a batch plan is large (~20 GB at B=11): keep the newest one, plus the B == 1 plan of the ort.run API path
            if B != 1:
                for k in [k for k in self._plans if k != 1]:
                    del self._plans[k]
            pl = _NetPlan(self, B)
            self._plans[B] = pl
        return pl

    # onnxruntime-compatible call (host arrays; API path used by MDX.process): input [B,4,dim_f,dim_t]
    @_ffi.on_device
    def run(self, _outputs, feed):
        x = torch.from_numpy(np.ascontiguousarray(feed["input"], dtype=np.float32)).to(self.device)
        B = x.shape[0]
        pl = self.plan(B)
        pl.spec_in.copy_(x.view(B, 2, 2, self.dim_f, self.dim_t).permute(0, 1, 4, 3, 2).reshape(B, 2, self.dim_t, 2 * self.dim_f))
        pl.run()
        y = pl.spec_out.view(B, 2, self.dim_t, self.dim_f, 2).permute(0, 1, 4, 3, 2).reshape(B, 4, self.dim_f, self.dim_t)
        return [y.cpu().numpy()]


class _NetPlan:
    """Buffers + prepared launches of the U-Net for a fixed chunk batch B.
    I/O in the DFT-friendly layout [B, ch, T, (f, ri)]; activations NHWC = [B, T, F, C]."""

    def __init__(self, net: ConvTDFNetB200, B: int):
        dev, W, be = net.device, net.W, net.backend
        R = be == tg.BACKEND_TC
        f32 = dict(device=dev, dtype=torch.float32)
        act = dict(device=dev, dtype=torch.float16 if net.half else torch.float32)   # activations inside the plan
        T, F, g, l, n, bnf = net.dim_t, net.dim_f, net.g, net.l, net.n, net.bn
        self.B = B
        steps: List = []
        add = steps.append
        self.spec_in = torch.empty(B, 2, T, 2 * F, **f32)
        self.spec_out = torch.empty(B, 2, T, 2 * F, **f32)
        max_elems = B * T * F * g
        pool = [torch.empty(max_elems, **act) for _ in range(3)]       # t1, t2, xt scratch shared by all levels

        def buf(slot, *shape):
            nel = 1
            for s_ in shape:
                nel *= s_
            return pool[slot][:nel].view(*shape)

        reps: Dict[str, torch.Tensor] = {}

        def rep(vec, rows_pc):
            """per-channel vector replicated over the (b,h) rows of the [B*H*C, W] TDF GEMMs."""
            return vec.repeat(rows_pc).contiguous()

        def tfc_tdf(x, key, Hh, Ww, c, out):
            """TFC (l 3x3 convs) + TDF (two bias-free linears along frequency, each BN + ReLU) + residual.  The TDF GEMMs
            run over rows (b, t, c) with K = frequency, i.e. on the NHCW transpose of the activations; both transposes
            live in GEMM epilogues (the last TFC conv also writes NHCW; the second TDF linear writes NHWC and adds the
            residual), so no standalone transpose pass touches HBM."""
            cur = x
            xt = buf(2, B, Hh, c, Ww)
            for j in range(l):
                dst = buf(j % 2, B, Hh, Ww, c)
                last = j == l - 1
                epi = Epi(bias=W[f"{key}.c{j}.b"], act_pre=tg.ACT_RELU, round_out=R and not last)
                if last:   # second output: the same values in NHCW order, RN-rounded for the TDF GEMM
                    epi.out2 = tg.Out(xt, Hh * c * Ww, c * Ww, 1, Hh, Ww, sn=Ww)
                    epi.round_out2 = R
                add(tg.conv2d(cur, W[f"{key}.c{j}.w"], dst, 3, 3, (1, 1), epi, be, name=f"{key}.c{j}"))
                cur = dst
            t = cur
            rows, Kb = B * Hh * c, Ww // bnf
            h = torch.empty(rows, Kb, device=dev, dtype=W[key + ".w2"].dtype)     # follows the operand type of the GEMM that reads it
            s1, b1 = rep(W[key + ".s1"], B * Hh), rep(W[key + ".b1"], B * Hh)
            s2, b2 = rep(W[key + ".s2"], B * Hh), rep(W[key + ".b2"], B * Hh)
            add(tg.linear(xt.view(rows, Ww), W[key + ".w1"], h,
                          Epi(row_scale_pre=s1, bias=b1, bias_per_row=True, act_pre=tg.ACT_RELU, row_scale=s2, round_out=R), be,
                          name=f"{key}.tdf1"))
            # rows tiled as (w = channel, h = (b, t)) so the epilogue can address NHWC: out[(b,t), n = f, c]
            bw = 1
            while bw < 128 and c % (2 * bw) == 0:
                bw *= 2
            a2 = tg.View(h, (Kb, c, B * Hh, 1, 1), (1, Kb, c * Kb, 0, 0))
            o2 = tg.Out(out, 0, Ww * c, 1, B * Hh, c, sn=c)
            add(tg.TapGemm(a2, tg.weights(W[key + ".w2"]), [(0, 0, 0, 0, 0)], (c, B * Hh, 1), o2,
                           Epi(bias=b2, bias_per_row=True, act_pre=tg.ACT_RELU, res=t, res_strides=(0, Ww * c, 1, c), round_out=R),
                           be, box=(bw, 128 // bw), name=f"{key}.tdf2"))

        # ---- first conv (1x1, 4 -> g) reading [B, ch, T, F, ri]: pointwise, write-bound -> its own row kernel
        x = torch.empty(B, T, F, g, **act)
        add(lambda x=x: ops.mdx_first_conv(self.spec_in, W["first.w4"], W["first.b"], x, R))
        Hh, Ww, c = T, F, g
        skips = []
        for i in range(n):
            y = torch.empty(B, Hh, Ww, c, **act)
            tfc_tdf(x, f"enc{i}", Hh, Ww, c, y)
            skips.append((y, Hh, Ww, c))
            x = torch.empty(B, Hh // 2, Ww // 2, c + g, **act)
            add(tg.conv2d_k2s2(y, W[f"ds{i}.w"], x, Epi(bias=W[f"ds{i}.b"], act_pre=tg.ACT_RELU, round_out=R), be, name=f"ds{i}"))
            Hh, Ww, c = Hh // 2, Ww // 2, c + g
        y = torch.empty(B, Hh, Ww, c, **act)
        tfc_tdf(x, "mid", Hh, Ww, c, y)
        x = y
        for i in range(n):
            sk, Hs, Ws, cs = skips[-1 - i]
            u = torch.empty(B, Hs, Ws, cs, **act)
            for op in tg.conv_transpose2d_k2s2(x, W[f"us{i}.w"], u,
                                               Epi(bias=W[f"us{i}.b"], act_pre=tg.ACT_RELU, res=sk, res_mul=True, res_mapped=True, round_out=R),
                                               be, name=f"us{i}"):
                add(op)
            Hh, Ww, c = Hs, Ws, cs
            y = torch.empty(B, Hh, Ww, c, **act)
            tfc_tdf(u, f"dec{i}", Hh, Ww, c, y)
            x = y
        # ---- final conv (1x1, g -> 4) writing [B, ch, T, F, ri]: pointwise, read-bound -> its own row kernel
        add(lambda x=x: ops.mdx_final_conv(x, W["final.w"], W["final.b"], self.spec_out, R))
        self.steps = steps
        self.graph = StepGraph(steps)

    def run(self):
        self.graph()


def shard_range(n_items: int, rank: int, world: int):
    """Contiguous share of `n_items` chunk inferences for `rank` of `world` (remainder to the low ranks)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_spans(n, n_fft, chunk_size, mt_threads, world, margin=44100):
    """For every rank of `world`: the half-open SAMPLE range [lo, hi) of the song its contiguous chunk range produces.
    Kept output samples are monotone in the flattened chunk order (half 0 keeps [0, n/2), half 1 keeps [n/2, n); inside a
    half chunk i keeps [i*gen, (i+1)*gen)), so a contiguous chunk range owns one contiguous slice of the stem — which is
    what makes the final concat an all-gather of disjoint slices (mdx.py:190-197, 107-117)."""
    src, lo, hi, dst, klo, khi = chunk_descriptors(n, n_fft, chunk_size, mt_threads, margin)
    gen = chunk_size - n_fft
    k_lo = np.maximum(dst, klo)
    k_hi = np.minimum(np.minimum(dst + gen, khi), n)
    spans = []
    for r in range(world):
        a, b = shard_range(len(src), r, world)
        live = [(int(k_lo[i]), int(k_hi[i])) for i in range(a, b) if k_hi[i] > k_lo[i]]
        spans.append((min(x for x, _ in live), max(y for _, y in live)) if live else (0, 0))
    return spans


def allgather_spans(t: torch.Tensor, spans, group) -> None:
    """In place: every rank holds valid data of t[:, lo_r:hi_r] for its own span and receives everybody else's.
    One all-gather of equal-size (padded) slices — the only collective of the sharded MDX pass."""
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    width = max(hi - lo for lo, hi in spans)
    if width == 0:
        return
    rows = t.shape[0]
    send = torch.zeros(rows, width, dtype=t.dtype, device=t.device)
    lo, hi = spans[rank]
    send[:, :hi - lo] = t[:, lo:hi]
    recv = torch.empty(world * rows, width, dtype=t.dtype, device=t.device)       # concatenation along dim 0 (gloo and nccl)
    dist.all_gather_into_tensor(recv, send, group=group)
    recv = recv.view(world, rows, width)
    for r, (lo, hi) in enumerate(spans):
        if r != rank and hi > lo:
            t[:, lo:hi] = recv[r, :, :hi - lo]


def segment_bounds(n, chunk_size, margin_size):
    """Start/end of the overlapping segments MDX.segment(combine=False) cuts (mdx.py:119-141)."""
    if chunk_size <= 0 or chunk_size > n:
        chunk_size = n
    if margin_size > chunk_size:
        margin_size = chunk_size
    bounds = []
    for count, skip in enumerate(range(0, n, chunk_size)):
        margin = 0 if count == 0 else margin_size
        end = min(skip + chunk_size + margin_size, n)
        bounds.append((skip - margin, end))
        if end == n:
            break
    return bounds


def chunk_descriptors(n, n_fft, chunk_size, mt_threads, margin=44100):
    """Flattens segment + pad_wave + trim + [:-pad] + segment(combine) (mdx.py:119-171, 195-197, 107-117) into one
    record per chunk inference: (src_start, lo, hi, dst_start, keep_lo, keep_hi), all in song sample coordinates.
    Chunk b reads song[src_start + s] for s in [0, chunk) where the index is inside [lo, hi) (zeros elsewhere) and its
    kept output sample k in [0, gen) lands at dst_start + k when that is inside [keep_lo, keep_hi)."""
    trim = n_fft // 2
    gen = chunk_size - 2 * trim
    bounds = segment_bounds(n, n // mt_threads, margin)
    src, lo, hi, dst, klo, khi = [], [], [], [], [], []
    for k, (a, b) in enumerate(bounds):
        nh = b - a
        pad = gen - nh % gen
        keep_lo = a + (0 if k == 0 else margin)                     # segment(combine=True) uses the default margin
        keep_hi = b - (0 if (k == len(bounds) - 1 or margin == 0) else margin)
        for i in range((nh + pad) // gen):
            src.append(a + i * gen - trim)
            lo.append(a)
            hi.append(b)
            dst.append(a + i * gen)
            klo.append(keep_lo)
            khi.append(keep_hi)
    return [np.asarray(v, dtype=np.int64) for v in (src, lo, hi, dst, klo, khi)]


class MDX:
    DEFAULT_SR = 44100
    DEFAULT_CHUNK_SIZE = 0 * DEFAULT_SR
    DEFAULT_MARGIN_SIZE = 1 * DEFAULT_SR
    DEFAULT_PROCESSOR = 0
    BATCH = 11          # chunks per network launch (a 4-min song is 2 x 22 chunks)

    def __init__(self, model_path, params: MDXModel, processor=DEFAULT_PROCESSOR, backend=tg.BACKEND_TC):
        if processor < 0:
            raise RuntimeError("b200vc MDX has no CPU execution provider")
        self.device = torch.device(f"cuda:{processor}")
        self.model = params
        sd = model_path if isinstance(model_path, dict) else load_mdx_weights(model_path, params.dim_t)
        if isinstance(sd, dict) and "state_dict" in sd:
            sd = sd["state_dict"]
        self.ort = ConvTDFNetB200(sd, self.device, backend)          # name kept from the reference (mdx.py:74)
        if (self.ort.dim_f, self.ort.dim_t) != (params.dim_f, params.dim_t):
            raise ValueError(f"network is {self.ort.dim_f}x{self.ort.dim_t} but MDXModel is {params.dim_f}x{params.dim_t}")
        self.backend = backend
        self.process = lambda spec: self.ort.run(None, {"input": spec.cpu().numpy()})[0]
        self.prog = None
        self._io = None
        self._desc_cache = {}

    @staticmethod
    def get_hash(model_path):
        """md5 of the last 10000 KiB of the file (whole file if shorter) — mdx.py:81-90."""
        try:
            with open(model_path, "rb") as f:
                f.seek(-10000 * 1024, 2)
                return hashlib.md5(f.read()).hexdigest()
        except OSError:
            with open(model_path, "rb") as f:
                return hashlib.md5(f.read()).hexdigest()

    @staticmethod
    def segment(wave, combine=True, chunk_size=DEFAULT_CHUNK_SIZE, margin_size=DEFAULT_MARGIN_SIZE):
        """Host arrays in/out exactly like mdx.py:92-141 (kept for API compatibility; the device path below
        folds the same index arithmetic into its chunk descriptors)."""
        if combine:
            out = None
            for i, seg in enumerate(wave):
                start = 0 if i == 0 else margin_size
                end = None if (i == len(wave) - 1 or margin_size == 0) else -margin_size
                out = seg[:, start:end] if out is None else np.concatenate((out, seg[:, start:end]), axis=-1)
            return out
        return [wave[:, a:b].copy() for (a, b) in MDX._segment_bounds(wave.shape[-1], chunk_size, margin_size)]

    @staticmethod
    def _segment_bounds(n, chunk_size, margin_size):
        return segment_bounds(n, chunk_size, margin_size)

    def _descriptors(self, n, mt_threads):
        m = self.model
        return chunk_descriptors(n, m.n_fft, m.chunk_size, mt_threads, self.DEFAULT_MARGIN_SIZE)

    @_ffi.on_device
    def _process_device(self, wave_dev: torch.Tensor, out_dev: torch.Tensor, sign: float, coef: float, accumulate: bool,
                        mt_threads: int, shard=(0, 1)):
        """Run this rank's share of the chunks of `sign * wave` through STFT -> net -> iSTFT and add coef * result into
        out_dev.  With shard=(rank, world) the flattened chunk list is split into contiguous ranges (chunks are
        independent, mdx.py:190-196); the caller sums the per-rank outputs (each sample is written by exactly one chunk)."""
        m, dev = self.model, self.device
        n = wave_dev.shape[1]
        # chunk descriptors of the whole sweep: built and uploaded ONCE per (song length, split, shard), padded to whole
        # batches with dummy chunks that read nothing (lo == hi) and keep nothing
        key = (n, mt_threads, tuple(shard))
        ent = self._desc_cache.get(key)
        if ent is None:
            desc = self._descriptors(n, mt_threads)
            c_lo, c_hi = shard_range(len(desc[0]), shard[0], shard[1])
            nchunks = c_hi - c_lo
            B = min(self.BATCH, max(nchunks, 1))
            padded_n = -(-nchunks // B) * B
            host = np.zeros((6, max(padded_n, 1)), dtype=np.int64)
            for r, v in enumerate(desc):
                host[r, :nchunks] = v[c_lo:c_hi]
            ent = (nchunks, B, torch.from_numpy(host).to(dev))
            if len(self._desc_cache) >= 8:
                self._desc_cache.pop(next(iter(self._desc_cache)))
            self._desc_cache[key] = ent
        nchunks, B, ddev = ent
        if nchunks == 0:
            return
        R = self.backend == tg.BACKEND_TC
        fwd, inv, env = m.dft(R)
        pl = self.ort.plan(B)
        if self._io is None or self._io[0] is not pl:      # keyed on the plan itself: a rebuilt plan owns new spec buffers
            half = m.n_fft // 2
            padded = torch.empty(B, 2, m.chunk_size + m.n_fft, device=dev)
            frames = torch.empty(B, 2, m.dim_t, m.n_fft, device=dev)
            stft = _stft_gemm(padded, fwd, pl.spec_in, m, self.backend)
            istft = tg.linear(pl.spec_out.view(-1, 2 * m.dim_f), inv, frames.view(-1, m.n_fft), None, self.backend, name="mdx.istft")
            # STFT -> U-Net -> iSTFT of one chunk batch as ONE replayable launch sequence (see plans.StepGraph)
            self._io = (pl, padded, frames, StepGraph([stft, *pl.steps, istft]))
        _, padded, frames, net_graph = self._io
        trim = m.n_fft // 2
        for s in range(0, nchunks, B):
            e = min(s + B, nchunks)
            d_src, d_lo, d_hi, d_dst, d_klo, d_khi = (ddev[r, s:s + B] for r in range(6))
            ops.mdx_gather_chunks(wave_dev, d_src, d_lo, d_hi, padded, m.chunk_size, trim, sign, R)
            net_graph()
            ops.mdx_ola_store(frames, env, d_dst, d_klo, d_khi, out_dev, m.dim_t, m.n_fft, m.hop, m.chunk_size, trim,
                              coef, accumulate)
            if self.prog is not None:
                self.prog.update(e - s)

    @_ffi.on_device
    def process_wave(self, wave: np.ndarray, mt_threads=1):
        """np [2,N] -> np [2,N] like mdx.py:201-235 (the thread count only decides the segment split here)."""
        w = torch.from_numpy(np.ascontiguousarray(wave, dtype=np.float32)).to(self.device)
        out = torch.zeros_like(w)
        self._process_device(w, out, 1.0, 1.0, False, mt_threads)
        return out.cpu().numpy()


def load_mdx_weights(path, dim_t: Optional[int] = None):
    """`.pt/.pth` state dict of the restated ConvTDFNet, or a UVR `.onnx` file decoded with the hand-rolled protobuf
    reader in onnx_io (what `ort.InferenceSession(model_path)` loads at mdx.py:74); `dim_t` (from model_data.json) is
    needed for `.onnx` because the graph is shape-agnostic along time."""
    if str(path).endswith(".onnx"):
        from .onnx_io import convtdfnet_state_dict
        if dim_t is None:
            raise ValueError(f"{path}: dim_t (2 ** mdx_dim_t_set of the model_data.json entry) is required for .onnx weights")
        return convtdfnet_state_dict(str(path), int(dim_t))
    return torch.load(path, map_location="cpu", weights_only=False)


def _read_wav_44k(filename):
    """librosa.load(filename, mono=False, sr=44100) replacement for WAV input (mdx.py:257)."""
    from math import gcd

    from scipy.signal import resample_poly

    sr, data = wavfile.read(filename)
    if data.dtype.kind == "i":
        data = data.astype(np.float32) / float(np.iinfo(data.dtype).max + 1)
    data = data.astype(np.float32)
    if data.ndim == 1:
        data = np.stack([data, data], 1)
    if sr != 44100:
        gg = gcd(int(sr), 44100)
        data = resample_poly(data, 44100 // gg, sr // gg, axis=0).astype(np.float32)
    return np.ascontiguousarray(data.T), 44100


def pcm16_soundfile(x: np.ndarray) -> np.ndarray:
    """float -> PCM_16 as `soundfile.write` does it (mdx.py:273,280: default subtype of .wav).  python-soundfile switches
    libsndfile's clipping ON for every file (SFC_SET_CLIPPING), which selects f2s_clip_array: scaled = x * 2^31 in float,
    >= 2^31 -> 0x7FFF, <= -2^31 -> -0x8000, else lrintf(scaled) >> 16 — i.e. floor(x * 32768) with saturation, not
    round(x * 32767).  The same conversion runs on the device for stems that stay in HBM (b200vc_pcm16_from_planar)."""
    s = np.asarray(x, dtype=np.float32) * np.float32(2147483648.0)
    with np.errstate(invalid="ignore"):
        q = (np.rint(s).astype(np.int64) >> 16)
    q = np.where(s >= np.float32(2147483648.0), 32767, np.where(s <= np.float32(-2147483648.0), -32768, q))
    return np.where(np.isnan(s), 0, q).astype(np.int16)


def _write_wav_pcm16(path, data_T, sr):
    wavfile.write(path, sr, pcm16_soundfile(data_T))


def run_mdx_device(mdx_sess: MDX, wave_dev: torch.Tensor, denoise=False, m_threads=2, group=None):
    """The arithmetic of run_mdx (mdx.py:257-280) on a device tensor [2,N]: returns (main, inverse) device tensors.
    NB the reference normalises `wave` in place by its peak and reuses the normalised array for the inverse stem."""
    with torch.cuda.device(mdx_sess.device):
        return _run_mdx_device(mdx_sess, wave_dev, denoise, m_threads, group)


def _run_mdx_device(mdx_sess: MDX, wave_dev: torch.Tensor, denoise, m_threads, group):
    model = mdx_sess.model
    peak = torch.maximum(wave_dev.max(), wave_dev.min().abs())       # max(np.max(w), abs(np.min(w))), kept on the device: no host sync
    w = (wave_dev / peak).contiguous()
    proc = torch.zeros_like(w)
    shard = (0, 1)
    if group is not None:
        import torch.distributed as dist
        shard = (dist.get_rank(group), dist.get_world_size(group))
    if denoise:
        mdx_sess._process_device(w, proc, -1.0, -0.5, False, m_threads, shard)      # -(P(-w)) * 0.5
        mdx_sess._process_device(w, proc, 1.0, 0.5, True, m_threads, shard)         # + P(w) * 0.5
    else:
        mdx_sess._process_device(w, proc, 1.0, 1.0, False, m_threads, shard)
    if shard[1] > 1:
        # the only collective on the path: every rank computed one contiguous, disjoint sample range of the stem (both
        # denoise sweeps use the same chunk split and were accumulated locally) -> all-gather of those slices over NVLink
        spans = shard_spans(w.shape[1], model.n_fft, model.chunk_size, m_threads, shard[1], MDX.DEFAULT_MARGIN_SIZE)
        allgather_spans(proc, spans, group)
    inverse = torch.empty_like(w)
    proc.mul_(peak)                                                   # wave_processed *= peak (mdx.py:267)
    ops.mdx_finalize(proc, w, inverse, 1.0, model.compensation)       # inverse = -proc * compensation + wave_norm (mdx.py:280)
    return proc, inverse


def run_mdx_arrays(mdx_sess: MDX, wave: np.ndarray, denoise=False, m_threads=2):
    """Host-array wrapper of run_mdx_device: returns (main [2,N], inverse [2,N]) float32."""
    w = torch.from_numpy(np.ascontiguousarray(wave, dtype=np.float32)).to(mdx_sess.device)
    proc, inverse = run_mdx_device(mdx_sess, w, denoise, m_threads)
    return proc.cpu().numpy(), inverse.cpu().numpy()


def run_mdx(model_params, output_dir, model_path, filename, exclude_main=False, exclude_inversion=False, suffix=None,
            invert_suffix=None, denoise=False, keep_orig=True, m_threads=2):
    """Same signature and outputs as mdx.run_mdx (mdx.py:238-287)."""
    if not torch.cuda.is_available():
        raise RuntimeError("b200vc: run_mdx needs a CUDA device (no CPU fallback)")
    device = torch.device("cuda:0")
    vram_gb = torch.cuda.get_device_properties(device).total_memory / 1024 ** 3
    m_threads = 1 if vram_gb < 8 else 2
    model_hash = MDX.get_hash(model_path)
    mp = model_params.get(model_hash)
    is_onnx = str(model_path).endswith(".onnx")
    if is_onnx and mp is None:
        raise KeyError(f"{model_path}: md5 tail {model_hash} is not in model_data.json (mdx.py:81-90)")
    weights = load_mdx_weights(model_path, 2 ** mp["mdx_dim_t_set"] if is_onnx else None)
    if mp is None and isinstance(weights, dict) and "params" in weights:
        mp = weights["params"]                      # synthetic checkpoints carry their own model_data entry
    model = MDXModel(device, dim_f=mp["mdx_dim_f_set"], dim_t=2 ** mp["mdx_dim_t_set"], n_fft=mp["mdx_n_fft_scale_set"],
                     stem_name=mp["primary_stem"], compensation=mp["compensate"])
    mdx_sess = MDX(weights, model)
    wave, sr = _read_wav_44k(filename)
    wave_processed, inverse = run_mdx_arrays(mdx_sess, wave, denoise, m_threads)
    stem_name = model.stem_name if suffix is None else suffix
    main_filepath = None
    base = os.path.basename(os.path.splitext(filename)[0])
    if not exclude_main:
        main_filepath = os.path.join(output_dir, f"{base}_{stem_name}.wav")
        _write_wav_pcm16(main_filepath, wave_processed.T, sr)
    invert_filepath = None
    if not exclude_inversion:
        diff_stem_name = stem_naming.get(stem_name) if invert_suffix is None else invert_suffix
        stem_name = f"{stem_name}_diff" if diff_stem_name is None else diff_stem_name
        invert_filepath = os.path.join(output_dir, f"{base}_{stem_name}.wav")
        _write_wav_pcm16(invert_filepath, inverse.T, sr)
    if not keep_orig:
        os.remove(filename)
    del mdx_sess, wave_processed, wave
    gc.collect()
    return main_filepath, invert_filepath
