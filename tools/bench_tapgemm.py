"""Micro-benchmark of the tap-GEMM kernels on representative hot-path shapes.
Usage (on the GPU box): python tools/bench_tapgemm.py [--simt]
Prints one line per shape: backend, ms, TFLOP/s, GB/s (algorithmic in+out bytes)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aicovergen_b200 import tapgemm as tg  # noqa: E402


WARM, ITERS = 3, 10
DT = torch.float32


def timeit(fn, warm=None, iters=None):
    warm = WARM if warm is None else warm
    iters = ITERS if iters is None else iters
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--simt", action="store_true")
    ap.add_argument("--out", default="gpurun_out/bench_tapgemm.jsonl")
    ap.add_argument("--only", default="", help="substring filter on the shape name")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warm", type=int, default=3)
    ap.add_argument("--fp16", action="store_true", help="fp16 operand / activation storage (wgmma f16)")
    args = ap.parse_args()
    global WARM, ITERS, DT
    DT = torch.float16 if args.fp16 else torch.float32
    WARM, ITERS = args.warm, args.iters
    backends = [("auto", tg.BACKEND_TC), ("tile", tg.BACKEND_TC_TILE), ("persist", tg.BACKEND_TC_V1)] + ([("simt", tg.BACKEND_SIMT)] if args.simt else [])
    if args.fp16:
        backends = [("auto", tg.BACKEND_TC), ("persist", tg.BACKEND_TC_V1)]
    shapes = [
        # name, T, Cin, Cout, k, dil
        ("voc.s1 C256 k3", 65980, 256, 256, 3, 1),
        ("voc.s1 C256 k11", 65980, 256, 256, 11, 5),
        ("voc.s2 C128 k7", 659800, 128, 128, 7, 3),
        ("voc.s3 C64 k7", 1319600, 64, 64, 7, 3),
        ("voc.s4 C32 k11", 2639200, 32, 32, 11, 1),
        ("hubert.ffn1", 3299, 768, 3072, 1, 1),
        ("hubert.ffn2", 3299, 3072, 768, 1, 1),
        ("encp.ffn1 k3", 6598, 192, 768, 3, 1),
        ("flow.wn k5", 6598, 192, 384, 5, 1),
        ("mdx.l0 c48 k3 (as 1d)", 786432, 48, 48, 9, 1),
        ("mdx.l2 c144 k3 (as 1d)", 49152, 144, 144, 9, 1),
    ]
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for name, T, Ci, Co, k, d in shapes:
            if args.only not in name:
                continue
            x = torch.randn(T, Ci, device="cuda").to(DT)
            w = (torch.randn(k, Co, Ci, device="cuda") / (Ci * k) ** 0.5).to(DT)
            b = torch.randn(Co, device="cuda")
            out = torch.empty(T, Co, device="cuda", dtype=DT)
            for bname, be in backends:
                op = tg.conv1d(x, w, out, dilation=d, epi=tg.Epi(bias=b, act_pre=tg.ACT_LRELU, act_pre_p=0.1), backend=be)
                ms = timeit(op)
                fl = 2.0 * T * Ci * Co * k
                by = x.element_size() * T * (Ci + Co)
                rec = dict(shape=name, backend=bname, ms=ms, tflops=fl / ms / 1e9, gbs=by / ms / 1e6)
                print(json.dumps(rec), flush=True)
                f.write(json.dumps(rec) + "\n")
        main2d(f, args.only)
        main_membound(f, args.only)


def main2d(f, only=""):
    """MDX-style 3x3 convolutions (NHWC), the layers that dominate the separation pass."""
    for name, B, H, W, C in [("mdx.l0 2d c48", 1, 256, 3072, 48), ("mdx.l0 2d c48 B4", 4, 256, 3072, 48), ("mdx.l1 2d c96", 1, 128, 1536, 96),
                             ("mdx.l1 2d c96 B4", 4, 128, 1536, 96), ("mdx.l2 2d c144 B4", 4, 64, 768, 144), ("mdx.l3 2d c192", 2, 32, 384, 192)]:
        if only not in name:
            continue
        x = torch.randn(B, H, W, C, device="cuda").to(DT)
        w = (torch.randn(9, C, C, device="cuda") / (9 * C) ** 0.5).to(DT)
        b = torch.randn(C, device="cuda")
        out = torch.empty(B, H, W, C, device="cuda", dtype=DT)
        for bname, be in [("auto", tg.BACKEND_TC), ("persist", tg.BACKEND_TC_V1)] + ([] if DT == torch.float16 else [("tile", tg.BACKEND_TC_TILE)]):
            op = tg.conv2d(x, w, out, 3, 3, (1, 1), tg.Epi(bias=b, act_pre=tg.ACT_RELU), backend=be)
            ms = timeit(op)
            fl = 2.0 * B * H * W * C * C * 9
            by = 2.0 * x.element_size() * B * H * W * C
            rec = dict(shape=name, backend=bname, ms=ms, tflops=fl / ms / 1e9, gbs=by / ms / 1e6, ws=op.ws_applicable())
            print(json.dumps(rec), flush=True)
            f.write(json.dumps(rec) + "\n")


def main_membound(f, only=""):
    """The residual-carrying, small-K layers of the MDX net (HBM-bound): k2s2 conv-transpose with the multiplicative skip,
    and the TDF output GEMM with the transposed store + residual."""
    if "us4" in only or not only:
        B, H, W, Ci, Co = 2, 128, 1536, 96, 48
        x = torch.randn(B, H, W, Ci, device="cuda").to(DT)
        w = (torch.randn(4, Co, Ci, device="cuda") / Ci ** 0.5).to(DT)
        b = torch.randn(Co, device="cuda")
        sk = torch.randn(B, 2 * H, 2 * W, Co, device="cuda").to(DT)
        out = torch.empty(B, 2 * H, 2 * W, Co, device="cuda", dtype=DT)
        for tag, epi in [("bias+relu+skip", tg.Epi(bias=b, act_pre=tg.ACT_RELU, res=sk, res_mul=True, res_mapped=True)),
                         ("bias+relu", tg.Epi(bias=b, act_pre=tg.ACT_RELU)), ("plain", tg.Epi())]:
            ops_ = tg.conv_transpose2d_k2s2(x, w, out, epi)
            ms = timeit(lambda: [o() for o in ops_])
            by = x.element_size() * (x.numel() * 2 + out.numel() * (2 if epi.res is not None else 1))
            rec = dict(shape=f"mdx.us4 k2s2 c96->48 [{tag}]", backend="auto", ms=ms, tflops=2.0 * B * H * W * Ci * Co * 4 / ms / 1e9, gbs=by / ms / 1e6)
            print(json.dumps(rec), flush=True)
            f.write(json.dumps(rec) + "\n")
    if "tdf2" in only or not only:
        BH, c, F_, Kb = 2 * 256, 48, 3072, 384
        h = torch.randn(BH * c, Kb, device="cuda").to(DT)
        w2 = (torch.randn(F_, Kb, device="cuda") / Kb ** 0.5).to(DT)
        b2 = torch.randn(BH * c, device="cuda")
        t = torch.randn(BH, F_, c, device="cuda").to(DT)
        out = torch.empty(BH, F_, c, device="cuda", dtype=DT)
        a2 = tg.View(h, (Kb, c, BH, 1, 1), (1, Kb, c * Kb, 0, 0))
        op = tg.TapGemm(a2, tg.weights(w2), [(0, 0, 0, 0, 0)], (c, BH, 1), tg.Out(out, 0, F_ * c, 1, BH, c, sn=c),
                        tg.Epi(bias=b2, bias_per_row=True, act_pre=tg.ACT_RELU, res=t, res_strides=(0, F_ * c, 1, c)), box=(16, 8))
        ms = timeit(op)
        by = h.element_size() * (h.numel() + 2 * out.numel())
        rec = dict(shape="mdx.tdf2 L0 (transposed store + residual)", backend="auto", ms=ms, tflops=2.0 * BH * c * Kb * F_ / ms / 1e9, gbs=by / ms / 1e6)
        print(json.dumps(rec), flush=True)
        f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
