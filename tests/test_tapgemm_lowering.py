"""Host logic: conv/linear -> tap-GEMM descriptor lowerings, checked on CPU with the
descriptor emulator (tests/emu.py) against torch.nn.functional."""
import torch
import torch.nn.functional as F

from aicovergen_b200 import tapgemm as tg
from emu import emulate

torch.manual_seed(0)


def close(a, b, tol=1e-4):
    err = (a - b).abs().max().item()
    ref = b.abs().max().item() + 1e-9
    assert err / ref < tol, (err, ref)


def test_linear_bias_act():
    x = torch.randn(300, 96)
    w = torch.randn(40, 96)
    b = torch.randn(40)
    out = torch.zeros(300, 40)
    op = tg.linear(x, w, out, tg.Epi(bias=b, act_pre=tg.ACT_LRELU, act_pre_p=0.1))
    emulate(op)
    close(out, F.leaky_relu(F.linear(x, w, b), 0.1))


def test_conv1d_dilated_residual_dual():
    T, Ci, Co, k, d = 257, 24, 24, 7, 3
    x = torch.randn(T, Ci)
    w = torch.randn(Co, Ci, k)
    b = torch.randn(Co)
    res = torch.randn(T, Co)
    out = torch.zeros(T, Co)
    out2 = torch.zeros(T, Co)
    op = tg.conv1d(x, tg.pack_conv1d(w), out, dilation=d,
                   epi=tg.Epi(bias=b, res=res, out2=out2, act2=tg.ACT_LRELU, act2_p=0.1))
    emulate(op)
    ref = F.conv1d(x.t()[None], w, b, dilation=d, padding=(k * d - d) // 2)[0].t() + res
    close(out, ref)
    close(out2, F.leaky_relu(ref, 0.1))


def test_conv1d_column_slice_io():
    # read a channel slice of a wider buffer, write into a slice of another
    T = 130
    xbuf = torch.randn(T, 48)
    obuf = torch.zeros(T, 64)
    w = torch.randn(16, 32, 3)
    op = tg.conv1d(xbuf[:, 8:40], tg.pack_conv1d(w), obuf[:, 16:32])
    emulate(op)
    ref = F.conv1d(xbuf[:, 8:40].t()[None], w, padding=1)[0].t()
    close(obuf[:, 16:32], ref)
    assert obuf[:, :16].abs().max() == 0 and obuf[:, 32:].abs().max() == 0


def test_conv1d_strided():
    for (k, s, pad) in [(3, 2, 0), (2, 2, 0), (10, 5, 0), (4, 2, 1), (8, 4, 2)]:
        T, Ci, Co = 40 * s, 8, 12
        x = torch.randn(T, Ci)
        w = torch.randn(Co, Ci, k)
        ref = F.conv1d(x.t()[None], w, stride=s, padding=pad)[0].t()
        out = torch.zeros(ref.shape[0], Co)
        op = tg.conv1d_strided(x, tg.pack_conv1d(w), out, stride=s, pad=pad)
        emulate(op)
        close(out, ref)


def test_conv_transpose1d():
    for (k, s) in [(16, 10), (4, 2), (20, 8), (24, 12), (16, 8), (16, 4)]:
        T, Ci, Co = 37, 16, 8
        p = (k - s) // 2
        x = torch.randn(T, Ci)
        w = torch.randn(Ci, Co, k)
        b = torch.randn(Co)
        ref = F.conv_transpose1d(x.t()[None], w, b, stride=s, padding=p)[0].t()
        out = torch.full((ref.shape[0], Co), float("nan"))
        for op in tg.conv_transpose1d(x, tg.pack_convt1d(w), out, s, p, tg.Epi(bias=b)):
            emulate(op)
        close(out, ref)


def test_conv2d_3x3_batch():
    B, H, W, Ci, Co = 2, 9, 16, 8, 12
    x = torch.randn(B, H, W, Ci)
    w = torch.randn(Co, Ci, 3, 3)
    b = torch.randn(Co)
    out = torch.zeros(B, H, W, Co)
    op = tg.conv2d(x, tg.pack_conv2d(w), out, 3, 3, (1, 1), tg.Epi(bias=b, act_pre=tg.ACT_RELU))
    emulate(op)
    ref = F.relu(F.conv2d(x.permute(0, 3, 1, 2), w, b, padding=1)).permute(0, 2, 3, 1)
    close(out, ref)


def test_conv_transpose2d_s2():
    B, H, W, Ci, Co = 1, 5, 8, 6, 4
    x = torch.randn(B, H, W, Ci)
    w = torch.randn(Ci, Co, 3, 3)
    ref = F.conv_transpose2d(x.permute(0, 3, 1, 2), w, stride=2, padding=1, output_padding=1).permute(0, 2, 3, 1)
    out = torch.full(ref.shape, float("nan"))
    for op in tg.conv_transpose2d_s2(x, tg.pack_convt2d(w), out, 3, 1):
        emulate(op)
    close(out, ref)
    # 2x2 stride 2 (MDX up-sampling)
    w2 = torch.randn(Ci, Co, 2, 2)
    ref = F.conv_transpose2d(x.permute(0, 3, 1, 2), w2, stride=2).permute(0, 2, 3, 1)
    out = torch.full(ref.shape, float("nan"))
    for op in tg.conv_transpose2d_s2(x, tg.pack_convt2d(w2), out, 2, 0):
        emulate(op)
    close(out, ref)


def test_conv2d_k2s2():
    B, H, W, Ci, Co = 2, 6, 8, 4, 5
    x = torch.randn(B, H, W, Ci)
    w = torch.randn(Co, Ci, 2, 2)
    out = torch.zeros(B, H // 2, W // 2, Co)
    op = tg.conv2d_k2s2(x, tg.pack_conv2d(w), out)
    emulate(op)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, stride=2).permute(0, 2, 3, 1)
    close(out, ref)


def test_bmm_nt_heads():
    T, H, D = 50, 3, 16
    q = torch.randn(T, H * D)
    k = torch.randn(T, H * D)
    # per-head views of [T, H*D] without copies
    qa = q.view(T, H, D).permute(1, 0, 2)
    ka = k.view(T, H, D).permute(1, 0, 2)
    Tp = 52
    sc = torch.zeros(H, T, Tp)
    op = tg.bmm_nt(qa, ka, sc[:, :, :T], tg.Epi(scale=0.25))
    emulate(op)
    ref = torch.einsum("htd,hsd->hts", qa, ka) * 0.25
    close(sc[:, :, :T], ref)
    # P @ V via V^T rows
    vt = torch.randn(H * D, Tp)
    vta = vt.view(H, D, Tp)[:, :, :T]
    o = torch.zeros(T, H * D)
    oa = o.view(T, H, D).permute(1, 0, 2)
    op2 = tg.bmm_nt(sc[:, :, :T], vta, oa)
    emulate(op2)
    close(oa, torch.einsum("hts,hds->htd", sc[:, :, :T], vta))


def test_bias_per_row_role_swap():
    # V^T = Wv @ X^T + b[:,None]
    T, Cc = 33, 24
    x = torch.randn(T, Cc)
    wv = torch.randn(20, Cc)
    b = torch.randn(20)
    out = torch.zeros(20, 36)
    op = tg.linear(wv, x, out[:, :T], tg.Epi(bias=b, bias_per_row=True))
    emulate(op)
    close(out[:, :T], (x @ wv.t() + b).t())


def _tdf_problem(B=2, H=5, W=24, C=16, bnf=4, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, C, generator=g)
    wc = torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5
    bc = torch.randn(C, generator=g)
    w1 = torch.randn(W // bnf, W, generator=g) / W ** 0.5
    w2 = torch.randn(W, W // bnf, generator=g) / (W // bnf) ** 0.5
    s1, b1, s2, b2 = (torch.randn(C, generator=g) for _ in range(4))
    t = F.relu(F.conv2d(x.permute(0, 3, 1, 2), wc, bc, padding=1))                 # [B,C,H,W]
    h = F.relu(F.linear(t, w1) * s1[None, :, None, None] + b1[None, :, None, None])
    y = F.relu(F.linear(h, w2) * s2[None, :, None, None] + b2[None, :, None, None])
    ref = (t + y).permute(0, 2, 3, 1).contiguous()                                 # NHWC
    return x, wc, bc, w1, w2, s1, b1, s2, b2, t, ref


def tdf_ops(x, wc, bc, w1, w2, s1, b1, s2, b2, backend=tg.BACKEND_TC, rnd=False):
    """The MDX-Net TFC->TDF->residual chain with both transposes inside GEMM epilogues (aicovergen_b200/mdx.py)."""
    B, H, W, C = x.shape
    Kb = w1.shape[0]
    kw = dict(device=x.device)
    t = torch.zeros(B, H, W, C, **kw)
    xt = torch.zeros(B, H, C, W, **kw)
    hbuf = torch.zeros(B * H * C, Kb, **kw)
    out = torch.zeros(B, H, W, C, **kw)
    rep = lambda v: v.repeat(B * H).contiguous()
    ops = [tg.conv2d(x, tg.pack_conv2d(wc) if wc.dim() == 4 else wc, t, 3, 3, (1, 1),
                     tg.Epi(bias=bc, act_pre=tg.ACT_RELU, out2=tg.Out(xt, H * C * W, C * W, 1, H, W, sn=W), round_out2=rnd), backend),
           tg.linear(xt.view(B * H * C, W), w1, hbuf,
                     tg.Epi(row_scale_pre=rep(s1), bias=rep(b1), bias_per_row=True, act_pre=tg.ACT_RELU, row_scale=rep(s2), round_out=rnd),
                     backend)]
    bw = 1
    while bw < 128 and C % (2 * bw) == 0:
        bw *= 2
    a2 = tg.View(hbuf, (Kb, C, B * H, 1, 1), (1, Kb, C * Kb, 0, 0))
    ops.append(tg.TapGemm(a2, tg.weights(w2), [(0, 0, 0, 0, 0)], (C, B * H, 1), tg.Out(out, 0, W * C, 1, B * H, C, sn=C),
                          tg.Epi(bias=rep(b2), bias_per_row=True, act_pre=tg.ACT_RELU, res=t, res_strides=(0, W * C, 1, C)),
                          backend, box=(bw, 128 // bw)))
    return ops, t, xt, out


def test_transposed_epilogues_tdf_chain():
    x, wc, bc, w1, w2, s1, b1, s2, b2, t_ref, ref = _tdf_problem()
    ops, t, xt, out = tdf_ops(x, wc, bc, w1, w2, s1, b1, s2, b2)
    for op in ops:
        emulate(op)
    close(t, t_ref.permute(0, 2, 3, 1))
    close(xt, t_ref.permute(0, 2, 1, 3))
    close(out, ref)


def test_conv_transpose2d_k2s2_two_gemms_with_mapped_skip():
    g = torch.Generator().manual_seed(5)
    B, H, W, Ci, Co = 2, 5, 7, 12, 8
    x = torch.randn(B, H, W, Ci, generator=g)
    w = torch.randn(Ci, Co, 2, 2, generator=g)
    b = torch.randn(Co, generator=g)
    sk = torch.randn(B, 2 * H, 2 * W, Co, generator=g)
    out = torch.zeros(B, 2 * H, 2 * W, Co)
    for op in tg.conv_transpose2d_k2s2(x, tg.pack_convt2d(w), out,
                                       tg.Epi(bias=b, act_pre=tg.ACT_RELU, res=sk, res_mul=True, res_mapped=True)):
        emulate(op)
    ref = F.relu(F.conv_transpose2d(x.permute(0, 3, 1, 2), w, b, stride=2)).permute(0, 2, 3, 1) * sk
    close(out, ref)


def test_fp16_tensors_descriptor_and_semantics():
    """fp16 operands / outputs / residual (b200vc.h `dtype`): flags, element-unit offsets and the same epilogue
    semantics, executed by the emulator on half tensors (the wgmma f16 path itself needs a GPU)."""
    g = torch.Generator().manual_seed(21)
    B, H, W, Ci, Co = 1, 6, 40, 48, 32
    x = torch.randn(B, H, W, Ci, generator=g).half()
    w = (torch.randn(Co, Ci, 3, 3, generator=g) / (9 * Ci) ** 0.5)
    b = torch.randn(Co, generator=g)
    res = torch.randn(B, H, W, Co, generator=g).half()
    out = torch.zeros(B, H, W, Co, dtype=torch.float16)
    out2 = torch.zeros(B, H, W, Co)                                   # second output stays fp32
    op = tg.conv2d(x, tg.pack_conv2d(w).half(), out, 3, 3, (1, 1), tg.Epi(bias=b, act_pre=tg.ACT_RELU, res=res, out2=out2))
    assert op.params.dtype == 1 | 2 | 8
    assert op.params.vec4 & 2 and op.params.vec4 & 16                 # 32 halfs per row = 64 bytes: still 16-byte aligned
    emulate(op)
    ref = F.relu(F.conv2d(x.float().permute(0, 3, 1, 2), w.half().float(), b, padding=1)).permute(0, 2, 3, 1) + res.float()
    close(out.float(), ref, 2e-3)
    close(out2, ref, 1e-5)
    # a column slice of a wider half buffer: offsets are in elements of the tensor's own type
    wide = torch.zeros(5, 96, dtype=torch.float16)
    lin = tg.linear(torch.randn(5, 64, generator=g).half(), torch.randn(32, 64, generator=g).half(), wide[:, 64:])
    assert lin.params.out == wide.data_ptr() + 2 * 64
