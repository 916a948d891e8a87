"""Host-side lowering of conv / linear / matmul layers onto the tap-GEMM C ABI.

Everything on the hot path that is a convolution, a linear layer or a batched
matmul is described by one `b200vc_tapgemm_params` (include/b200vc.h) and run by
`b200vc_tapgemm` on either the wgmma TF32 / fp16 kernels or the exact-fp32 SIMT
kernel.  This module only builds descriptors (pure index arithmetic, testable on
CPU against torch.nn.functional with tests/emu.py); it never computes.

Layouts: activations channels-last ([T, C] / [H, W, C] / [B, H, W, C]);
weights packed per tap as [ntaps, N, K] (K contiguous).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional, Sequence, Tuple

import torch

from . import _ffi
from ._ffi import (ACT_EXP, ACT_GELU, ACT_LRELU, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH,
                   BACKEND_SIMT, BACKEND_TC, BACKEND_TC_TILE, BACKEND_TC_V1, BACKEND_TC_WS, MAX_TAPS, TapGemmParams)

__all__ = [
    "View", "Weights", "Out", "Epi", "TapGemm", "view", "out_of",
    "linear", "conv1d", "conv1d_strided", "conv_transpose1d", "conv2d", "conv_transpose2d_s2",
    "conv2d_k2s2", "bmm_nt",
    "pack_conv1d", "pack_convt1d", "pack_conv2d", "pack_convt2d",
    "ACT_NONE", "ACT_RELU", "ACT_LRELU", "ACT_GELU", "ACT_TANH", "ACT_SIGMOID", "ACT_EXP",
    "BACKEND_SIMT", "BACKEND_TC", "BACKEND_TC_V1", "BACKEND_TC_TILE", "BACKEND_TC_WS", "conv_transpose2d_k2s2",
]


# ---------------------------------------------------------------------------
# descriptors
# ---------------------------------------------------------------------------
@dataclass
class View:
    """Rank-5 strided read view (c, w, h, b, p) over tensor `t` starting `off` elements in."""
    t: torch.Tensor
    dims: Tuple[int, int, int, int, int]
    strides: Tuple[int, int, int, int, int]
    off: int = 0

    def ptr(self) -> int:
        return self.t.data_ptr() + self.t.element_size() * self.off


def view(x: torch.Tensor) -> View:
    """View of a channels-last tensor [W,C] / [H,W,C] / [B,H,W,C] (stride(-1) must be 1)."""
    assert x.dtype in (torch.float32, torch.float16) and x.stride(-1) == 1, (x.dtype, x.stride())
    shp, st = list(x.shape), list(x.stride())
    while len(shp) < 4:
        shp.insert(0, 1)
        st.insert(0, 0)
    B, H, W, Cc = shp
    sb, sh, sw, _ = st
    return View(x, (Cc, W, H, B, 1), (1, sw, sh, sb, 0))


@dataclass
class Weights:
    """Weight slices W[widx, n, k]: element at t[off + k + n*ldw + widx*wstride]."""
    t: torch.Tensor
    K: int
    N: int
    ldw: int
    wstride: int
    off: int = 0

    def ptr(self) -> int:
        return self.t.data_ptr() + self.t.element_size() * self.off


def weights(w: torch.Tensor) -> Weights:
    """Packed weights [ntaps, N, K] (or [N, K]) contiguous."""
    assert w.dtype in (torch.float32, torch.float16) and w.is_contiguous()
    if w.dim() == 2:
        w = w.unsqueeze(0)
    nt, N, K = w.shape
    return Weights(w, K, N, K, N * K)


@dataclass
class Out:
    """Output addressing: element (b,h,w,n) at t[off + b*sb + (h*osh+ooh)*sh + (w*osw+oow)*sw + n*sn]
    (sn = 1: channels-last; anything else writes a transposed layout)."""
    t: torch.Tensor
    sb: int
    sh: int
    sw: int
    fh: int
    fw: int
    off: int = 0
    osh: int = 1
    osw: int = 1
    ooh: int = 0
    oow: int = 0
    sn: int = 1

    def ptr(self) -> int:
        return self.t.data_ptr() + self.t.element_size() * self.off


def out_of(x: torch.Tensor, **kw) -> Out:
    """Output spec writing a channels-last tensor [W,N] / [H,W,N] / [B,H,W,N] (may be a column slice)."""
    assert x.dtype in (torch.float32, torch.float16) and x.stride(-1) == 1
    shp, st = list(x.shape), list(x.stride())
    while len(shp) < 4:
        shp.insert(0, 1)
        st.insert(0, 0)
    B, H, W, _ = shp
    sb, sh, sw, _ = st
    return Out(x, sb, sh, sw, H, W, **kw)


@dataclass
class Epi:
    """Fused epilogue: v=acc*row_scale_pre+bias; v=act_pre(v); v*=row_scale; v(+|*)=res; v*=scale; v+=res2;
    v=act_post(v); out=v; out2=act2(v)."""
    row_scale_pre: Optional[torch.Tensor] = None   # [OH*OW] per-output-row multiplier applied to the accumulator
    bias: Optional[torch.Tensor] = None
    bias_per_row: bool = False
    act_pre: int = ACT_NONE
    act_pre_p: float = 0.0
    row_scale: Optional[torch.Tensor] = None   # [OH*OW] per-output-row multiplier applied after act_pre
    res: Optional[torch.Tensor] = None     # channels-last tensor over the output pixel space
    res_mul: bool = False                  # v *= res instead of v += res
    res_mapped: bool = False               # address res by the mapped output pixel (conv-transpose phases)
    res_strides: Optional[Tuple[int, int, int, int]] = None   # explicit (sb, sh, sw, sn) element strides of `res`
    scale: float = 1.0
    res2: Optional[torch.Tensor] = None    # same addressing as out
    act_post: int = ACT_NONE
    act_post_p: float = 0.0
    out2: Optional[object] = None          # Tensor: same addressing as out; Out: its own (possibly transposed) layout
    act2: int = ACT_NONE
    act2_p: float = 0.0
    round_out: bool = False     # store `out` rounded (RN) to TF32: for tensors only consumed by TF32 GEMMs
    round_out2: bool = False
    split_out: int = 0          # > 0: write `out` as 3xTF32 planes hi | lo | hi, `split_out` elements apart (b200vc.h `split`)
    res_split: int = 0          # > 0: `res` is a split tensor, value = res[..] + res[.. + res_split]
    acc_in: Optional[torch.Tensor] = None   # fp32 partial sums [.., N] channels-last over the GEMM pixel space, added to the accumulator


def _tile_box(OW: int, OH: int) -> Tuple[int, int]:
    bw = 1
    while bw < OW and bw < 128:
        bw *= 2
    return bw, 128 // bw


class TapGemm:
    """A prepared launch. Holds the ctypes descriptor and keeps every tensor alive."""

    def __init__(self, a: View, w: Weights, taps: Sequence[Tuple[int, int, int, int, int]],
                 out_space: Tuple[int, int, int], out: Out, epi: Optional[Epi] = None,
                 backend: int = BACKEND_TC, w_batch_step: int = 0, Kc: Optional[int] = None,
                 N: Optional[int] = None, box: Optional[Tuple[int, int]] = None, name: str = ""):
        epi = epi or Epi()
        self.a, self.w, self.out, self.epi = a, w, out, epi
        self.taps = list(taps)
        self.name = name
        assert 1 <= len(self.taps) <= MAX_TAPS, len(self.taps)
        OW, OH, OB = out_space
        p = TapGemmParams()
        p.A = a.ptr()
        for i in range(5):
            p.a_dim[i] = int(a.dims[i])
            p.a_stride[i] = int(a.strides[i])
        assert a.strides[0] == 1
        p.Wt = w.ptr()
        p.ldw, p.wstride = int(w.ldw), int(w.wstride)
        p.w_batch_step = int(w_batch_step)
        p.Kc = int(Kc if Kc is not None else w.K)
        p.N = int(N if N is not None else w.N)
        p.ntaps = len(self.taps)
        p.OW, p.OH, p.OB = int(OW), int(OH), int(OB)
        bw, bh = box if box is not None else _tile_box(OW, OH)
        assert bw * bh == 128
        p.BW, p.BH = bw, bh
        p.osh, p.osw, p.ooh, p.oow = out.osh, out.osw, out.ooh, out.oow
        p.o_fh, p.o_fw = int(out.fh), int(out.fw)
        p.o_sb, p.o_sh, p.o_sw, p.o_sn = int(out.sb), int(out.sh), int(out.sw), int(out.sn)
        p.r_sn = 1
        self._keep = [a.t, w.t, out.t]
        if a.t.is_cuda:     # launches use the current device's stream (see _ffi.on_device); CPU tensors = descriptor emulator tests
            assert a.t.device == w.t.device == out.t.device and a.t.device.index == torch.cuda.current_device(), \
                f"tapgemm[{name}]: operands on {a.t.device}/{w.t.device}/{out.t.device}, current device cuda:{torch.cuda.current_device()}"
        # ---- epilogue
        if epi.row_scale_pre is not None:
            assert epi.row_scale_pre.dtype == torch.float32 and epi.row_scale_pre.is_contiguous()
            p.row_scale_pre = epi.row_scale_pre.data_ptr()
            self._keep.append(epi.row_scale_pre)
        if epi.bias is not None:
            assert epi.bias.dtype == torch.float32 and epi.bias.is_contiguous()
            p.bias = epi.bias.data_ptr()
            self._keep.append(epi.bias)
        p.bias_per_row = int(epi.bias_per_row)
        p.act_pre, p.act_pre_p = epi.act_pre, float(epi.act_pre_p)
        if epi.row_scale is not None:
            assert epi.row_scale.dtype == torch.float32 and epi.row_scale.is_contiguous()
            p.row_scale = epi.row_scale.data_ptr()
            self._keep.append(epi.row_scale)
        p.r_sb = p.r_sh = p.r_sw = 0
        if epi.res is not None:
            r = epi.res
            assert r.dtype in (torch.float32, torch.float16)
            if epi.res_strides is not None:
                p.r_sb, p.r_sh, p.r_sw, p.r_sn = (int(v_) for v_ in epi.res_strides)
            else:
                assert r.stride(-1) == 1
                st = list(r.stride())
                while len(st) < 4:
                    st.insert(0, 0)
                p.r_sb, p.r_sh, p.r_sw = int(st[0]), int(st[1]), int(st[2])
            p.res = r.data_ptr()
            p.res_op = (1 if epi.res_mul else 0) | (2 if epi.res_mapped else 0)
            self._keep.append(r)
        p.scale = float(epi.scale)
        if epi.res2 is not None:
            assert epi.res2.stride() == out.t.stride() or epi.res2.shape == out.t.shape
            p.res2 = epi.res2.data_ptr() + epi.res2.element_size() * out.off
            self._keep.append(epi.res2)
        p.act_post, p.act_post_p = epi.act_post, float(epi.act_post_p)
        p.out = out.ptr()
        if isinstance(epi.out2, Out):
            o2 = epi.out2
            p.out2 = o2.ptr()
            p.out2_own = 1
            p.o2_sb, p.o2_sh, p.o2_sw, p.o2_sn = int(o2.sb), int(o2.sh), int(o2.sw), int(o2.sn)
            self._keep.append(o2.t)
        elif epi.out2 is not None:
            assert epi.out2.stride() == out.t.stride()
            p.out2 = epi.out2.data_ptr() + epi.out2.element_size() * out.off
            self._keep.append(epi.out2)
        p.act2, p.act2_p = epi.act2, float(epi.act2_p)
        p.round_tf32 = (1 if epi.round_out else 0) | (2 if epi.round_out2 else 0)
        p.split = (1 if epi.split_out else 0) | (2 if epi.res_split else 0)
        p.o_split, p.r_split = int(epi.split_out), int(epi.res_split)
        if epi.split_out:
            assert epi.res2 is None and epi.out2 is None and out.t.dtype == torch.float32 and out.sn == 1
            assert epi.split_out % 4 == 0
        if epi.res_split:
            assert epi.res is not None and epi.res.dtype == torch.float32 and epi.res_split % 4 == 0
        if epi.acc_in is not None:
            ai = epi.acc_in
            assert ai.dtype == torch.float32 and ai.stride(-1) == 1 and ai.data_ptr() % 16 == 0
            st = list(ai.stride())
            while len(st) < 4:
                st.insert(0, 0)
            assert all(s_ % 4 == 0 for s_ in st[:3])
            p.acc_in = ai.data_ptr()
            p.ai_sb, p.ai_sh, p.ai_sw = int(st[0]), int(st[1]), int(st[2])
            self._keep.append(ai)
        for i, (c_off, dw, dh, dp, widx) in enumerate(self.taps):
            t = p.taps[i]
            t.c_off, t.dw, t.dh, t.dp, t.widx = int(c_off), int(dw), int(dh), int(dp), int(widx)
        # ---- element types: fp16 operands / epilogue tensors (tensor-core backends only; see b200vc.h `dtype`)
        half = torch.float16
        assert a.t.dtype == w.t.dtype, "A and W must have the same element type"
        dt = 1 if a.t.dtype == half else 0
        dt |= 2 if out.t.dtype == half else 0
        o2t = epi.out2.t if isinstance(epi.out2, Out) else epi.out2
        dt |= 4 if (o2t is not None and o2t.dtype == half) else 0
        dt |= 8 if (epi.res is not None and epi.res.dtype == half) else 0
        dt |= 16 if (epi.res2 is not None and epi.res2.dtype == half) else 0
        p.dtype = dt
        es_a = a.t.element_size()
        es_o, es_o2 = out.t.element_size(), (o2t.element_size() if o2t is not None else 4)
        es_r = epi.res.element_size() if epi.res is not None else 4
        es_r2 = epi.res2.element_size() if epi.res2 is not None else 4
        # ---- vectorisation flags (16-byte alignment of base pointers and of every stride, in bytes)
        v = 0
        k_ok = dt == 0 and (p.A or 0) % 16 == 0 and (p.Wt or 0) % 16 == 0 and p.ldw % 4 == 0 and p.wstride % 4 == 0
        k_ok = k_ok and all(a.dims[i] <= 1 or a.strides[i] % 4 == 0 for i in range(1, 5))
        k_ok = k_ok and all(t[0] % 4 == 0 for t in self.taps)
        if k_ok:
            v |= 1

        def al(ptr, es, *strides):
            return (ptr or 0) % 16 == 0 and all((s_ * es) % 16 == 0 for s_ in strides)

        shared2 = p.out2 if not p.out2_own else 0
        if p.o_sn == 1 and al(p.out, es_o, p.o_sb, p.o_sh, p.o_sw) and al(shared2, es_o2, p.o_sb, p.o_sh, p.o_sw) and \
                al(p.res2, es_r2, p.o_sb, p.o_sh, p.o_sw):
            v |= 2
        if al(p.bias, 4) or p.bias_per_row:
            v |= 4
        if not p.out2_own or (p.o2_sn == 1 and al(p.out2, es_o2, p.o2_sb, p.o2_sh, p.o2_sw)):
            v |= 8
        if not p.res or (p.r_sn == 1 and al(p.res, es_r, p.r_sb, p.r_sh, p.r_sw)):
            v |= 16
        p.vec4 = v
        self.params = p
        self.backend = backend
        self._tc_ok = None

    # ------------------------------------------------------------------
    def tc_supported(self) -> bool:
        if self._tc_ok is None:
            self._tc_ok = bool(_ffi.lib().b200vc_tapgemm_tc_supported(C.byref(self.params)))
        return self._tc_ok

    def ws_applicable(self) -> bool:
        return bool(_ffi.lib().b200vc_tapgemm_ws_applicable(C.byref(self.params)))

    def flops(self) -> int:
        p = self.params
        return 2 * p.OW * p.OH * p.OB * p.N * p.Kc * p.ntaps

    def __call__(self, stream: Optional[int] = None, backend: Optional[int] = None):
        be = self.backend if backend is None else backend
        if be in (BACKEND_TC, BACKEND_TC_V1, BACKEND_TC_TILE) and not self.tc_supported():
            if self.params.dtype:
                raise ValueError(f"tapgemm[{self.name}]: fp16 tensors need a TMA-addressable problem (tensor-core kernels only)")
            be = BACKEND_SIMT   # operand not TMA-addressable (e.g. C==1); still CUDA, still fp32-exact
        if stream is None:
            stream = torch.cuda.current_stream().cuda_stream
        rc = _ffi.lib().b200vc_tapgemm(C.byref(self.params), be, C.c_void_p(stream))
        if rc != 0:
            _ffi.check(rc, f"tapgemm[{self.name}]")


# ---------------------------------------------------------------------------
# weight packing (done once at model load)
# ---------------------------------------------------------------------------
def pack_conv1d(w: torch.Tensor) -> torch.Tensor:
    """torch Conv1d weight [Cout, Cin, k] -> [k, Cout, Cin]."""
    return w.permute(2, 0, 1).contiguous().float()


def pack_convt1d(w: torch.Tensor) -> torch.Tensor:
    """torch ConvTranspose1d weight [Cin, Cout, k] -> [k, Cout, Cin]."""
    return w.permute(2, 1, 0).contiguous().float()


def pack_conv2d(w: torch.Tensor) -> torch.Tensor:
    """torch Conv2d weight [Cout, Cin, kh, kw] -> [kh*kw, Cout, Cin]."""
    co, ci, kh, kw = w.shape
    return w.permute(2, 3, 0, 1).reshape(kh * kw, co, ci).contiguous().float()


def pack_convt2d(w: torch.Tensor) -> torch.Tensor:
    """torch ConvTranspose2d weight [Cin, Cout, kh, kw] -> [kh*kw, Cout, Cin]."""
    ci, co, kh, kw = w.shape
    return w.permute(2, 3, 1, 0).reshape(kh * kw, co, ci).contiguous().float()


# ---------------------------------------------------------------------------
# lowerings
# ---------------------------------------------------------------------------
def linear(x: torch.Tensor, w: torch.Tensor, out: torch.Tensor, epi: Optional[Epi] = None,
           backend: int = BACKEND_TC, name: str = "linear") -> TapGemm:
    """out[..., n] = sum_k x[..., k] w[n, k]  (x: [T,K] / [H,W,K] / [B,H,W,K] channels-last)."""
    a = view(x)
    W = weights(w)
    o = out_of(out)
    return TapGemm(a, W, [(0, 0, 0, 0, 0)], (a.dims[1], a.dims[2], a.dims[3]), o, epi, backend, name=name)


def conv1d(x: torch.Tensor, wp: torch.Tensor, out: torch.Tensor, dilation: int = 1,
           pad: Optional[int] = None, epi: Optional[Epi] = None, backend: int = BACKEND_TC,
           name: str = "conv1d") -> TapGemm:
    """Stride-1 Conv1d. x [T,Cin] (or [B,T,Cin]), wp [k,Cout,Cin] packed, out [T_out,Cout]."""
    k = wp.shape[0]
    if pad is None:
        pad = (k * dilation - dilation) // 2
    a = view(x) if x.dim() == 2 else _view_bt(x)
    o = out_of(out) if out.dim() == 2 else _out_bt(out)
    taps = [(0, j * dilation - pad, 0, 0, j) for j in range(k)]
    return TapGemm(a, weights(wp), taps, (o.fw, 1, a.dims[3]), o, epi, backend, name=name)


def _view_bt(x: torch.Tensor) -> View:
    B, T, Cc = x.shape
    return View(x, (Cc, T, 1, B, 1), (1, x.stride(1), 0, x.stride(0), 0))


def _out_bt(x: torch.Tensor) -> Out:
    B, T, _ = x.shape
    return Out(x, x.stride(0), 0, x.stride(1), 1, T)


def conv1d_strided(x: torch.Tensor, wp: torch.Tensor, out: torch.Tensor, stride: int, pad: int = 0,
                   epi: Optional[Epi] = None, backend: int = BACKEND_TC,
                   name: str = "conv1d_s") -> TapGemm:
    """Strided Conv1d via the [T/s, s*C] reshape view. x [T,Cin] with T % stride == 0 and
    row pitch == Cin (contiguous rows); tap j reads row floor((j-pad)/s), channel block (j-pad) mod s."""
    T, Cin = x.shape
    assert T % stride == 0 and x.stride(0) == Cin and x.stride(1) == 1
    k = wp.shape[0]
    a = View(x, (stride * Cin, T // stride, 1, 1, 1), (1, stride * Cin, 0, 0, 0))
    taps = []
    for j in range(k):
        pos = j - pad
        taps.append(((pos % stride) * Cin, pos // stride, 0, 0, j))
    o = out_of(out)
    return TapGemm(a, weights(wp), taps, (o.fw, 1, 1), o, epi, backend, name=name)


def conv_transpose1d(x: torch.Tensor, wp: torch.Tensor, out: torch.Tensor, stride: int, padding: int,
                     epi: Optional[Epi] = None, backend: int = BACKEND_TC, name: str = "convT1d"):
    """ConvTranspose1d as `stride` phase GEMMs. x [T,Cin], wp [k,Cout,Cin] (pack_convt1d), out [T*stride,Cout].
    Output o = i*stride + j - padding; phase r = (o + padding) mod stride uses taps j = r + stride*m."""
    T, _ = x.shape
    k = wp.shape[0]
    a = view(x)
    ops = []
    for r in range(stride):
        taps = [(0, -m, 0, 0, r + stride * m) for m in range((k - r + stride - 1) // stride) if r + stride * m < k]
        if not taps:
            continue
        o = out_of(out, osw=stride, oow=r - padding)
        ops.append(TapGemm(a, weights(wp), taps, (T + (k - 1) // stride, 1, 1), o, epi, backend,
                           name=f"{name}.ph{r}"))
    return ops


def conv2d(x: torch.Tensor, wp: torch.Tensor, out: torch.Tensor, kh: int, kw: int, pad: Tuple[int, int],
           epi: Optional[Epi] = None, backend: int = BACKEND_TC, name: str = "conv2d") -> TapGemm:
    """Stride-1 Conv2d. x [B,H,W,Cin] (or [H,W,Cin]); wp [kh*kw,Cout,Cin]; out [B,H,W,Cout]."""
    a = view(x)
    o = out_of(out)
    taps = [(0, dx - pad[1], dy - pad[0], 0, dy * kw + dx) for dy in range(kh) for dx in range(kw)]
    return TapGemm(a, weights(wp), taps, (o.fw, o.fh, a.dims[3]), o, epi, backend, name=name)


def conv_transpose2d_s2(x: torch.Tensor, wp: torch.Tensor, out: torch.Tensor, k: int, pad: int,
                        epi: Optional[Epi] = None, backend: int = BACKEND_TC, name: str = "convT2d",
                        stride: Tuple[int, int] = (2, 2)):
    """ConvTranspose2d (square kernel k, padding pad, per-axis stride 1 or 2) as phase GEMMs.
    x [B,H,W,Cin]; wp [k*k,Cout,Cin] (pack_convt2d); out [B,H*sh,W*sw,Cout]."""
    a = view(x)
    B, H, W = a.dims[3], a.dims[2], a.dims[1]
    sh_, sw_ = stride
    ops = []
    for ry in range(sh_):
        ty = [(m, ry + sh_ * m) for m in range(k) if ry + sh_ * m < k]
        for rx in range(sw_):
            tx = [(m, rx + sw_ * m) for m in range(k) if rx + sw_ * m < k]
            taps = [(0, -mx, -my, 0, jy * k + jx) for (my, jy) in ty for (mx, jx) in tx]
            if not taps:
                continue
            o = out_of(out, osh=sh_, osw=sw_, ooh=ry - pad, oow=rx - pad)
            ops.append(TapGemm(a, weights(wp), taps, (W + (k - 1) // sw_, H + (k - 1) // sh_, B), o, epi,
                               backend, name=f"{name}.ph{ry}{rx}"))
    return ops


def conv_transpose2d_k2s2(x: torch.Tensor, wp: torch.Tensor, out: torch.Tensor, epi: Optional[Epi] = None,
                          backend: int = BACKEND_TC, name: str = "convT2d_k2s2"):
    """ConvTranspose2d(kernel 2, stride 2, no padding) as TWO GEMMs (one per output row parity) with N = 2*Cout:
    the outputs for column parities 0/1 of one input pixel are adjacent in NHWC memory, so they form one 2*Cout-wide
    GEMM row written at pixel stride 2*Cout.  Half the input reads and twice the MMA width of the 4-phase form.
    x [B,H,W,Cin]; wp [4,Cout,Cin] (pack_convt2d); out [B,2H,2W,Cout] contiguous.  A mapped residual (MDX-Net skip)
    and a per-column bias are re-addressed for the widened rows here."""
    import dataclasses
    a = view(x)
    B, H, W = a.dims[3], a.dims[2], a.dims[1]
    four, Cout, Cin = wp.shape
    assert four == 4 and wp.is_contiguous() and tuple(out.shape) == (B, 2 * H, 2 * W, Cout) and out.stride(-1) == 1
    assert out.stride(2) == Cout, "output pixels must be densely packed"
    e2 = dataclasses.replace(epi) if epi is not None else Epi()
    assert e2.res2 is None and e2.out2 is None and e2.row_scale is None and e2.row_scale_pre is None
    if e2.bias is not None and not e2.bias_per_row:
        e2.bias = torch.cat([e2.bias, e2.bias]).contiguous()
    if e2.res is not None:
        assert e2.res_mapped and tuple(e2.res.shape) == tuple(out.shape) and e2.res.stride(-1) == 1 and e2.res.stride(2) == Cout
        st = e2.res.stride()
        e2.res_strides = (st[0], st[1], 2 * st[2], 1)
    ops = []
    for ry in range(2):
        w2 = Weights(wp, Cin, 2 * Cout, Cin, 2 * Cout * Cin, off=ry * 2 * Cout * Cin)
        o = Out(out, out.stride(0), out.stride(1), 2 * out.stride(2), 2 * H, W, osh=2, ooh=ry)
        ops.append(TapGemm(a, w2, [(0, 0, 0, 0, 0)], (W, H, B), o, e2, backend, name=f"{name}.ph{ry}"))
    return ops


def conv2d_k2s2(x: torch.Tensor, wp: torch.Tensor, out: torch.Tensor, epi: Optional[Epi] = None,
                backend: int = BACKEND_TC, name: str = "conv2d_k2s2") -> TapGemm:
    """2x2 stride-2 Conv2d (no padding) through a rank-5 view: (2C, W/2, H/2, B, dy).
    x [B,H,W,C] contiguous with H,W even; wp [4,Cout,C]; out [B,H/2,W/2,Cout]."""
    if x.dim() == 3:
        x = x.unsqueeze(0)
    B, H, W, Cc = x.shape
    assert H % 2 == 0 and W % 2 == 0 and x.is_contiguous()
    a = View(x, (2 * Cc, W // 2, H // 2, B, 2), (1, 2 * Cc, 2 * W * Cc, H * W * Cc, W * Cc))
    taps = [(dx * Cc, 0, 0, dy, dy * 2 + dx) for dy in range(2) for dx in range(2)]
    o = out_of(out)
    return TapGemm(a, weights(wp), taps, (W // 2, H // 2, B), o, epi, backend, Kc=Cc, name=name)


def bmm_nt(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, epi: Optional[Epi] = None,
           backend: int = BACKEND_TC, name: str = "bmm") -> TapGemm:
    """Batched out[g] = a[g] @ b[g]^T with a [G,M,K], b [G,N,K], out [G,M,N]; arbitrary
    (4-element aligned) batch/row strides, unit stride along K and along out's N."""
    G, M, K = a.shape
    G2, N, K2 = b.shape
    assert G == G2 and K == K2 and a.stride(2) == 1 and b.stride(2) == 1 and out.stride(2) == 1
    av = View(a, (K, M, 1, G, 1), (1, a.stride(1), 0, a.stride(0), 0))
    W = Weights(b, K, N, b.stride(1), b.stride(0))
    o = Out(out, out.stride(0), 0, out.stride(1), 1, M)
    return TapGemm(av, W, [(0, 0, 0, 0, 0)], (M, 1, G), o, epi, backend, w_batch_step=1, name=name)
