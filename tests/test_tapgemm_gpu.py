"""GPU parity of the tap-GEMM kernels (SIMT fp32 and wgmma TF32 / fp16) through the C ABI,
against torch CPU fp32 convolutions on the same seeded inputs."""
import pytest
import torch
import torch.nn.functional as F

from aicovergen_b200 import _ffi
from aicovergen_b200 import tapgemm as tg

pytestmark = pytest.mark.gpu

BACKENDS = [("simt", tg.BACKEND_SIMT, 2e-5), ("tc", tg.BACKEND_TC, 2e-3), ("tile", tg.BACKEND_TC_TILE, 2e-3),
            ("persist", tg.BACKEND_TC_V1, 2e-3)]


def rel_rms(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).pow(2).mean().sqrt() / (b.pow(2).mean().sqrt() + 1e-12)).item()


def check(out, ref, tol, what):
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    e = rel_rms(out, ref)
    mx = (out.cpu() - ref).abs().max().item()
    print(f"[tapgemm] {what}: rel_rms={e:.3e} max_abs={mx:.3e}")
    assert e < tol, f"{what}: rel rms {e} >= {tol} (max abs {mx})"


def dev(*ts):
    return [t.cuda() for t in ts]


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
@pytest.mark.parametrize("T,K,N", [(1000, 192, 384), (128, 32, 32), (4097, 768, 192), (300, 48, 48), (513, 100, 360)])
def test_linear(bname, backend, tol, T, K, N):
    g = torch.Generator().manual_seed(T + K + N)
    x = torch.randn(T, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = F.gelu(F.linear(x, w, b))
    xd, wd, bd = dev(x, w, b)
    out = torch.full((T, N), float("nan"), device="cuda")
    tg.linear(xd, wd, out, tg.Epi(bias=bd, act_pre=tg.ACT_GELU), backend=backend)()
    torch.cuda.synchronize()
    check(out, ref, tol, f"linear[{bname}] T{T} K{K} N{N}")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
@pytest.mark.parametrize("C,k,d", [(32, 11, 5), (64, 7, 3), (128, 3, 1), (256, 3, 5), (192, 5, 1)])
def test_conv1d_resblock_style(bname, backend, tol, C, k, d):
    g = torch.Generator().manual_seed(C * 100 + k * 10 + d)
    T = 3001
    x = torch.randn(T, C, generator=g)
    w = torch.randn(C, C, k, generator=g) / (C * k) ** 0.5
    b = torch.randn(C, generator=g)
    res = torch.randn(T, C, generator=g)
    ref = F.conv1d(x.t()[None], w, b, dilation=d, padding=(k * d - d) // 2)[0].t() + res
    xd, wd, bd, rd = dev(x, tg.pack_conv1d(w), b, res)
    out = torch.full((T, C), float("nan"), device="cuda")
    out2 = torch.full((T, C), float("nan"), device="cuda")
    tg.conv1d(xd, wd, out, dilation=d, epi=tg.Epi(bias=bd, res=rd, out2=out2, act2=tg.ACT_LRELU, act2_p=0.1),
              backend=backend)()
    torch.cuda.synchronize()
    check(out, ref, tol, f"conv1d[{bname}] C{C} k{k} d{d}")
    check(out2, F.leaky_relu(ref, 0.1), tol, f"conv1d.out2[{bname}] C{C} k{k} d{d}")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
def test_conv1d_inplace_accumulate(bname, backend, tol):
    g = torch.Generator().manual_seed(5)
    T, C = 700, 64
    x = torch.randn(T, C, generator=g)
    w = torch.randn(C, C, 3, generator=g) / (C * 3) ** 0.5
    acc0 = torch.randn(T, C, generator=g)
    ref = F.leaky_relu((F.conv1d(x.t()[None], w, padding=1)[0].t() + x) / 3 + acc0, 0.1)
    xd, wd = dev(x, tg.pack_conv1d(w))
    accd = acc0.cuda()
    tg.conv1d(xd, wd, accd, epi=tg.Epi(res=xd, scale=1 / 3, res2=accd, act_post=tg.ACT_LRELU, act_post_p=0.1),
              backend=backend)()
    torch.cuda.synchronize()
    check(accd, ref, tol, f"conv1d.inplace[{bname}]")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
@pytest.mark.parametrize("k,s,Ci,Co", [(3, 2, 512, 512), (2, 2, 512, 512), (10, 5, 64, 96)])
def test_conv1d_strided(bname, backend, tol, k, s, Ci, Co):
    g = torch.Generator().manual_seed(k * 7 + s)
    T = 400 * s
    x = torch.randn(T, Ci, generator=g)
    w = torch.randn(Co, Ci, k, generator=g) / (Ci * k) ** 0.5
    ref = F.gelu(F.conv1d(x.t()[None], w, stride=s)[0].t())
    xd, wd = dev(x, tg.pack_conv1d(w))
    out = torch.full((ref.shape[0], Co), float("nan"), device="cuda")
    tg.conv1d_strided(xd, wd, out, s, 0, tg.Epi(act_pre=tg.ACT_GELU), backend=backend)()
    torch.cuda.synchronize()
    check(out, ref, tol, f"conv1d_strided[{bname}] k{k} s{s}")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
@pytest.mark.parametrize("k,s,Ci,Co", [(16, 10, 512, 256), (16, 10, 256, 128), (4, 2, 128, 64), (4, 2, 64, 32), (24, 12, 64, 32)])
def test_conv_transpose1d(bname, backend, tol, k, s, Ci, Co):
    g = torch.Generator().manual_seed(k + s + Ci)
    T, p = 211, (k - s) // 2
    x = torch.randn(T, Ci, generator=g)
    w = torch.randn(Ci, Co, k, generator=g) / (Ci * k / s) ** 0.5
    b = torch.randn(Co, generator=g)
    ref = F.conv_transpose1d(x.t()[None], w, b, stride=s, padding=p)[0].t()
    xd, wd, bd = dev(x, tg.pack_convt1d(w), b)
    out = torch.full((ref.shape[0], Co), float("nan"), device="cuda")
    for op in tg.conv_transpose1d(xd, wd, out, s, p, tg.Epi(bias=bd), backend=backend):
        op()
    torch.cuda.synchronize()
    check(out, ref, tol, f"convT1d[{bname}] k{k} s{s} {Ci}->{Co}")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
@pytest.mark.parametrize("B,H,W,Ci,Co", [(1, 64, 128, 16, 16), (2, 33, 32, 64, 128), (1, 96, 4, 256, 512), (1, 40, 256, 48, 96),
                                        (2, 21, 384, 48, 48), (1, 9, 200, 64, 32)])
def test_conv2d_3x3(bname, backend, tol, B, H, W, Ci, Co):
    g = torch.Generator().manual_seed(H + W + Ci)
    x = torch.randn(B, H, W, Ci, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5
    b = torch.randn(Co, generator=g)
    res = torch.randn(B, H, W, Co, generator=g)
    ref = (F.relu(F.conv2d(x.permute(0, 3, 1, 2), w, b, padding=1)).permute(0, 2, 3, 1) + res).contiguous()
    xd, wd, bd, rd = dev(x, tg.pack_conv2d(w), b, res)
    out = torch.full((B, H, W, Co), float("nan"), device="cuda")
    tg.conv2d(xd, wd, out, 3, 3, (1, 1), tg.Epi(bias=bd, act_pre=tg.ACT_RELU, res=rd), backend=backend)()
    torch.cuda.synchronize()
    check(out, ref, tol, f"conv2d[{bname}] {B}x{H}x{W} {Ci}->{Co}")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
def test_conv2d_concat_slices(bname, backend, tol):
    """Producer writes into a channel slice of a concat buffer; consumer reads the full buffer."""
    g = torch.Generator().manual_seed(11)
    H, W, Cc = 32, 64, 32
    x = torch.randn(1, H, W, Cc, generator=g)
    skip = torch.randn(1, H, W, Cc, generator=g)
    w1 = torch.randn(Cc, Cc, 3, 3, generator=g) / (Cc * 9) ** 0.5
    w2 = torch.randn(Cc, 2 * Cc, 3, 3, generator=g) / (2 * Cc * 9) ** 0.5
    y1 = F.conv2d(x.permute(0, 3, 1, 2), w1, padding=1)
    ref = F.conv2d(torch.cat([y1, skip.permute(0, 3, 1, 2)], 1), w2, padding=1).permute(0, 2, 3, 1).contiguous()
    cat = torch.full((1, H, W, 2 * Cc), float("nan"), device="cuda")
    cat[..., Cc:] = skip.cuda()
    xd, w1d, w2d = dev(x, tg.pack_conv2d(w1), tg.pack_conv2d(w2))
    tg.conv2d(xd, w1d, cat[..., :Cc], 3, 3, (1, 1), backend=backend)()
    out = torch.full((1, H, W, Cc), float("nan"), device="cuda")
    tg.conv2d(cat, w2d, out, 3, 3, (1, 1), backend=backend)()
    torch.cuda.synchronize()
    check(out, ref, tol * 2, f"conv2d.concat[{bname}]")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
def test_conv_transpose2d_and_k2s2(bname, backend, tol):
    g = torch.Generator().manual_seed(3)
    B, H, W, Ci, Co = 1, 24, 16, 64, 32
    x = torch.randn(B, H, W, Ci, generator=g)
    w = torch.randn(Ci, Co, 3, 3, generator=g) / (Ci * 2.25) ** 0.5
    ref = F.conv_transpose2d(x.permute(0, 3, 1, 2), w, stride=2, padding=1, output_padding=1).permute(0, 2, 3, 1).contiguous()
    xd, wd = dev(x, tg.pack_convt2d(w))
    out = torch.full(tuple(ref.shape), float("nan"), device="cuda")
    for op in tg.conv_transpose2d_s2(xd, wd, out, 3, 1, backend=backend):
        op()
    torch.cuda.synchronize()
    check(out, ref, tol, f"convT2d[{bname}]")
    w2 = torch.randn(Co, Ci, 2, 2, generator=g) / (Ci * 4) ** 0.5
    ref2 = F.conv2d(x.permute(0, 3, 1, 2), w2, stride=2).permute(0, 2, 3, 1).contiguous()
    out2 = torch.full(tuple(ref2.shape), float("nan"), device="cuda")
    tg.conv2d_k2s2(xd, tg.pack_conv2d(w2).cuda(), out2, backend=backend)()
    torch.cuda.synchronize()
    check(out2, ref2, tol, f"conv2d_k2s2[{bname}]")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
def test_attention_matmuls(bname, backend, tol):
    g = torch.Generator().manual_seed(9)
    T, Hh, D = 777, 12, 64
    Tp = (T + 3) // 4 * 4
    q = torch.randn(T, Hh * D, generator=g)
    k = torch.randn(T, Hh * D, generator=g)
    vt = torch.randn(Hh * D, Tp, generator=g)
    qa = q.view(T, Hh, D).permute(1, 0, 2)
    ka = k.view(T, Hh, D).permute(1, 0, 2)
    ref_s = torch.einsum("htd,hsd->hts", qa, ka) * 0.125
    qd, kd, vtd = dev(q, k, vt)
    sc = torch.zeros(Hh, T, Tp, device="cuda")
    tg.bmm_nt(qd.view(T, Hh, D).permute(1, 0, 2), kd.view(T, Hh, D).permute(1, 0, 2), sc[:, :, :T],
              tg.Epi(scale=0.125), backend=backend)()
    torch.cuda.synchronize()
    check(sc[:, :, :T], ref_s, tol, f"qk^T[{bname}]")
    p = torch.softmax(ref_s, -1)
    pd = torch.zeros(Hh, T, Tp, device="cuda")
    pd[:, :, :T] = p.cuda()
    o = torch.full((T, Hh * D), float("nan"), device="cuda")
    tg.bmm_nt(pd[:, :, :T], vtd.view(Hh, D, Tp)[:, :, :T], o.view(T, Hh, D).permute(1, 0, 2), backend=backend)()
    torch.cuda.synchronize()
    ref_o = torch.einsum("hts,hds->htd", p, vt.view(Hh, D, Tp)[:, :, :T]).permute(1, 0, 2).reshape(T, Hh * D)
    check(o, ref_o, tol, f"pv[{bname}]")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
def test_overlapping_frames_dft(bname, backend, tol):
    """STFT-as-GEMM: A rows are overlapping frames (row stride = hop < n_fft)."""
    g = torch.Generator().manual_seed(21)
    n_fft, hop, nfr, nb = 1024, 160, 300, 64
    sig = torch.randn(hop * (nfr - 1) + n_fft, generator=g)
    basis = torch.randn(nb, n_fft, generator=g) / n_fft ** 0.5
    frames = sig.unfold(0, n_fft, hop)
    ref = frames @ basis.t()
    sd, bd = dev(sig, basis)
    out = torch.full((nfr, nb), float("nan"), device="cuda")
    a = tg.View(sd, (n_fft, nfr, 1, 1, 1), (1, hop, 0, 0, 0))
    tg.TapGemm(a, tg.weights(bd), [(0, 0, 0, 0, 0)], (nfr, 1, 1), tg.out_of(out), backend=backend)()
    torch.cuda.synchronize()
    check(out, ref, tol, f"dft-frames[{bname}]")


def test_weight_stationary_kernel_is_selected_and_forced():
    """Small-channel regular convolutions qualify for tapgemm_ws.cu; forcing it on a non-qualifying descriptor errors."""
    x = torch.randn(1000, 64, device="cuda")
    w = torch.randn(7, 64, 64, device="cuda")
    out = torch.empty(1000, 64, device="cuda")
    op = tg.conv1d(x, w, out, dilation=3)
    assert op.ws_applicable()
    op(backend=tg.BACKEND_TC_WS)
    torch.cuda.synchronize()
    big = tg.conv1d(torch.randn(1000, 256, device="cuda"), torch.randn(3, 256, 256, device="cuda"), torch.empty(1000, 256, device="cuda"))
    assert not big.ws_applicable()
    with pytest.raises(RuntimeError):
        big(backend=tg.BACKEND_TC_WS)


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
@pytest.mark.parametrize("B,H,W,C,bnf", [(2, 5, 24, 16, 4), (1, 16, 256, 48, 8), (2, 8, 128, 96, 8), (1, 4, 64, 40, 4)])
def test_transposed_epilogues_tdf_chain(bname, backend, tol, B, H, W, C, bnf):
    """conv -> (NHWC, NHCW) dual store; TDF linears over (b,t,c) rows; NHWC store + residual from the transposed GEMM."""
    from test_tapgemm_lowering import _tdf_problem, tdf_ops
    x, wc, bc, w1, w2, s1, b1, s2, b2, t_ref, ref = _tdf_problem(B, H, W, C, bnf, seed=B + H + W + C)
    args = dev(x, tg.pack_conv2d(wc), bc, w1, w2, s1, b1, s2, b2)
    ops, t, xt, out = tdf_ops(*args, backend=backend)
    for op in ops:
        op()
    torch.cuda.synchronize()
    check(t, t_ref.permute(0, 2, 3, 1).contiguous(), tol, f"tfc[{bname}]")
    check(xt, t_ref.permute(0, 2, 1, 3).contiguous(), tol, f"tfc^T[{bname}]")
    check(out, ref, 2 * tol, f"tdf[{bname}]")


@pytest.mark.parametrize("bname,backend,tol", BACKENDS)
@pytest.mark.parametrize("B,H,W,Ci,Co", [(2, 5, 7, 12, 8), (1, 16, 192, 96, 48), (2, 8, 64, 288, 240)])
def test_conv_transpose2d_k2s2_two_gemms(bname, backend, tol, B, H, W, Ci, Co):
    g = torch.Generator().manual_seed(Ci + Co)
    x = torch.randn(B, H, W, Ci, generator=g)
    w = torch.randn(Ci, Co, 2, 2, generator=g) / Ci ** 0.5
    b = torch.randn(Co, generator=g)
    sk = torch.randn(B, 2 * H, 2 * W, Co, generator=g)
    ref = (F.relu(F.conv_transpose2d(x.permute(0, 3, 1, 2), w, b, stride=2)).permute(0, 2, 3, 1) * sk).contiguous()
    xd, wd, bd, sd = dev(x, tg.pack_convt2d(w), b, sk)
    out = torch.full((B, 2 * H, 2 * W, Co), float("nan"), device="cuda")
    for op in tg.conv_transpose2d_k2s2(xd, wd, out, tg.Epi(bias=bd, act_pre=tg.ACT_RELU, res=sd, res_mul=True, res_mapped=True),
                                       backend=backend):
        op()
    torch.cuda.synchronize()
    check(out, ref, tol, f"convT k2s2[{bname}]")


@pytest.mark.parametrize("T,Ci,Co,k", [(50000, 64, 160, 3), (41000, 96, 96, 5), (45000, 32, 48, 3), (70001, 32, 32, 1)])
def test_persistent_256_row_tiles_conv1d(T, Ci, Co, k):
    """(experimental path, enabled through b200vc_tapgemm_set_rows256)
    Problems with >= #SM 256-row tiles take the path of the persistent kernel where one B tile feeds two 128-row blocks
    (BN <= 128; BN 256 keeps 128-row tiles); checked against the exact-fp32 SIMT kernel on the same device."""
    g = torch.Generator().manual_seed(T)
    x, w, b = torch.randn(T, Ci, generator=g), torch.randn(Co, Ci, k, generator=g) / (Ci * k) ** 0.5, torch.randn(Co, generator=g)
    res = torch.randn(T, Co, generator=g)
    xd, wd, bd, rd = dev(x, tg.pack_conv1d(w), b, res)
    outs = []
    _ffi.lib().b200vc_tapgemm_set_rows256(1)
    try:
        for be in (tg.BACKEND_SIMT, tg.BACKEND_TC_V1):
            o = torch.full((T, Co), float("nan"), device="cuda")
            tg.conv1d(xd, wd, o, dilation=2, epi=tg.Epi(bias=bd, act_pre=tg.ACT_LRELU, act_pre_p=0.1, res=rd), backend=be)()
            outs.append(o)
        torch.cuda.synchronize()
    finally:
        _ffi.lib().b200vc_tapgemm_set_rows256(0)
    check(outs[1].cpu(), outs[0].cpu(), 2e-3, f"persistent 256-row tiles T={T} {Ci}->{Co} k{k}")


def test_persistent_256_row_tiles_conv2d():
    g = torch.Generator().manual_seed(9)
    B, H, W, Ci, Co = 2, 72, 384, 48, 96            # box (16 x 8) doubled along h -> 16 x 16
    x = torch.randn(B, H, W, Ci, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5
    b = torch.randn(Co, generator=g)
    xd, wd, bd = dev(x, tg.pack_conv2d(w), b)
    outs = []
    _ffi.lib().b200vc_tapgemm_set_rows256(1)
    try:
        for be in (tg.BACKEND_SIMT, tg.BACKEND_TC_V1):
            o = torch.full((B, H, W, Co), float("nan"), device="cuda")
            tg.conv2d(xd, wd, o, 3, 3, (1, 1), tg.Epi(bias=bd, act_pre=tg.ACT_RELU), backend=be)()
            outs.append(o)
        torch.cuda.synchronize()
    finally:
        _ffi.lib().b200vc_tapgemm_set_rows256(0)
    check(outs[1].cpu(), outs[0].cpu(), 2e-3, "persistent 256-row tiles conv2d")


# ------------------------------------------------------------------------------------------------------------------
# fp16 operand storage (wgmma f16): the default storage of the MDX-Net U-Net from round 2 on.
# ------------------------------------------------------------------------------------------------------------------
import os  # noqa: E402

experimental = pytest.mark.gpu          # (was an opt-in marker in round 1)


@experimental
@pytest.mark.parametrize("backend", [tg.BACKEND_TC, tg.BACKEND_TC_V1])
@pytest.mark.parametrize("T,Ci,Co,k,d", [(3000, 128, 128, 3, 1), (5000, 64, 64, 7, 3), (2500, 48, 96, 3, 1), (777, 768, 384, 1, 1)])
def test_fp16_conv1d(backend, T, Ci, Co, k, d):
    g = torch.Generator().manual_seed(T + Ci)
    x = torch.randn(T, Ci, generator=g).half()
    w = (torch.randn(Co, Ci, k, generator=g) / (Ci * k) ** 0.5).half()
    b = torch.randn(Co, generator=g)
    res = torch.randn(T, Co, generator=g).half()
    ref = F.leaky_relu(F.conv1d(x.float().t()[None], w.float(), b, dilation=d, padding=(k * d - d) // 2)[0].t(), 0.1) + res.float()
    xd, wd, bd, rd = dev(x, tg.pack_conv1d(w.float()).half(), b, res)
    out = torch.full((T, Co), float("nan"), device="cuda", dtype=torch.float16)
    out2 = torch.full((T, Co), float("nan"), device="cuda")
    tg.conv1d(xd, wd, out, dilation=d, epi=tg.Epi(bias=bd, act_pre=tg.ACT_LRELU, act_pre_p=0.1, res=rd, out2=out2), backend=backend)()
    torch.cuda.synchronize()
    check(out2.cpu(), ref, 2e-3, f"fp16 conv1d fp32 out2 T={T} {Ci}->{Co}")
    check(out.float().cpu(), ref, 3e-3, f"fp16 conv1d half out T={T} {Ci}->{Co}")


@experimental
@pytest.mark.parametrize("B,H,W,Ci,Co", [(1, 40, 256, 48, 48), (2, 21, 384, 48, 96), (1, 16, 128, 144, 144)])
def test_fp16_conv2d(B, H, W, Ci, Co):
    g = torch.Generator().manual_seed(H + W)
    x = torch.randn(B, H, W, Ci, generator=g).half()
    w = (torch.randn(Co, Ci, 3, 3, generator=g) / (Ci * 9) ** 0.5).half()
    b = torch.randn(Co, generator=g)
    ref = F.relu(F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, padding=1)).permute(0, 2, 3, 1).contiguous()
    xd, wd, bd = dev(x, tg.pack_conv2d(w.float()).half(), b)
    out = torch.full((B, H, W, Co), float("nan"), device="cuda", dtype=torch.float16)
    tg.conv2d(xd, wd, out, 3, 3, (1, 1), tg.Epi(bias=bd, act_pre=tg.ACT_RELU))()
    torch.cuda.synchronize()
    check(out.float().cpu(), ref, 3e-3, f"fp16 conv2d {Ci}->{Co}")
