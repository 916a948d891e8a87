"""The MDX U-Net launch plan (aicovergen_b200/mdx.py: _NetPlan) executed on CPU: every tap-GEMM through the descriptor
emulator, the two pointwise row kernels through torch.  Checks, without a GPU, that the plan computes the oracle's network
and — for the fp16-storage mode — that every GEMM in it is addressable by the TMA/wgmma kernels (the fp16 path has no
SIMT fallback)."""
import pytest
import torch

import aicovergen_b200.mdx as bm
from aicovergen_b200 import ops
from aicovergen_b200 import tapgemm as tg
from aicovergen_b200.synthetic import make_mdx_state_dict
from emu import emulate
from oracle import mdx as om


def _first_conv(spec, w4, bias, out, round_out=False):
    B, T, F, g = out.shape
    x = spec.view(B, 2, T, F, 2).permute(0, 2, 3, 1, 4).reshape(B, T, F, 4)        # (ch0re, ch0im, ch1re, ch1im)
    out.copy_(torch.relu(x @ w4.t() + bias).to(out.dtype))


def _final_conv(x, w, bias, spec, round_out=False):
    B, T, F, c = x.shape
    y = x.float() @ w.t() + bias                                                    # [B,T,F,4]
    spec.copy_(y.view(B, T, F, 2, 2).permute(0, 3, 1, 2, 4).reshape(B, 2, T, 2 * F))


def _run_plan_on_cpu(net, x, monkeypatch):
    monkeypatch.setattr(ops, "mdx_first_conv", _first_conv)
    monkeypatch.setattr(ops, "mdx_final_conv", _final_conv)
    B = x.shape[0]
    pl = bm._NetPlan(net, B)
    pl.spec_in.copy_(x.view(B, 2, 2, net.dim_f, net.dim_t).permute(0, 1, 4, 3, 2).reshape(B, 2, net.dim_t, 2 * net.dim_f))
    gemms = []
    for st in pl.steps:
        if isinstance(st, tg.TapGemm):
            gemms.append(st)
            emulate(st)
        else:
            st()
    y = pl.spec_out.view(B, 2, net.dim_t, net.dim_f, 2).permute(0, 1, 4, 3, 2).reshape(B, 4, net.dim_f, net.dim_t)
    return y, gemms


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("cfg", [dict(dim_f=64, dim_t=16, g=8, l=2, n=2, bn=4), dict(dim_f=96, dim_t=8, g=16, l=1, n=1, bn=4)])
def test_mdx_plan_matches_oracle_on_cpu(cfg, half, monkeypatch):
    monkeypatch.setattr(bm, "MDX_FP16", half)
    sd = make_mdx_state_dict(**cfg)
    net = bm.ConvTDFNetB200(sd, "cpu", tg.BACKEND_TC)
    assert net.half == half
    x = torch.randn(2, 4, cfg["dim_f"], cfg["dim_t"], generator=torch.Generator().manual_seed(3)) * 2.0
    got, gemms = _run_plan_on_cpu(net, x, monkeypatch)
    ref = om.convtdfnet(sd, x)
    err = float((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
    assert torch.isfinite(got).all() and err < (8e-3 if half else 2e-3), err       # fp32 mode: weights are TF32-rounded
    n_half = 0
    for op in gemms:
        if op.params.dtype & 1:
            n_half += 1
            assert op.tc_supported(), f"{op.name}: fp16 operands but not TMA-addressable"
    if half:
        assert n_half >= len(gemms) - 2 * (cfg["n"] * 2 + 1)      # at most the K-misaligned TDF GEMMs stay fp32
    else:
        assert n_half == 0


@pytest.mark.parametrize("geom", [dict(dim_f=3072, dim_t=256, g=48), dict(dim_f=2048, dim_t=256, g=32)])
def test_full_size_fp16_plan_is_tma_addressable(geom, monkeypatch):
    """Descriptors only (no arithmetic): at the real UVR geometries every fp16 GEMM of the plan satisfies the TMA alignment
    rules, and only the bottleneck-level TDF output GEMM (K pitch 24 B) keeps fp32 operands."""
    monkeypatch.setattr(bm, "MDX_FP16", True)
    sd = make_mdx_state_dict(n=5, **geom)
    net = bm.ConvTDFNetB200(sd, "cpu", tg.BACKEND_TC)
    pl = bm._NetPlan(net, 1)
    gemms = [st for st in pl.steps if isinstance(st, tg.TapGemm)]
    fp32_ops = [op.name for op in gemms if not (op.params.dtype & 1)]
    for op in gemms:
        if op.params.dtype & 1:
            assert op.tc_supported(), op.name
    assert all(name.endswith("tdf2") for name in fp32_ops) and len(fp32_ops) <= 3, fp32_ops


def test_calibrated_batchnorm_keeps_stored_activations_in_fp16_range(monkeypatch):
    """synthetic.calibrate_mdx_batchnorm gives a synthetic net the activation statistics of a trained one: outputs stay
    O(1), the fp16-storage plan (emulated) then matches the oracle as closely as the TF32 path does."""
    from aicovergen_b200.synthetic import calibrate_mdx_batchnorm

    cfg = dict(dim_f=64, dim_t=16, g=8, l=2, n=2, bn=4)
    g = torch.Generator().manual_seed(11)
    sd = calibrate_mdx_batchnorm(make_mdx_state_dict(**cfg), torch.randn(2, 4, 64, 16, generator=g) * 30.0)
    x = torch.randn(2, 4, 64, 16, generator=g) * 30.0                 # another draw of the same (large) scale
    ref = om.convtdfnet(sd, x)
    assert float(ref.abs().max()) < 50.0
    monkeypatch.setattr(bm, "MDX_FP16", True)
    net = bm.ConvTDFNetB200(sd, "cpu", tg.BACKEND_TC)
    got, gemms = _run_plan_on_cpu(net, x, monkeypatch)
    err = float((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
    assert torch.isfinite(got).all() and err < 8e-3, err
    for op in gemms:                                                  # every stored fp16 tensor stayed finite and small
        if op.params.dtype & 2:
            assert float(op.out.t.float().abs().max()) < 1e3, op.name


def test_vocoder_fp16_resblock_plan_is_tma_addressable(monkeypatch):
    """Opt-in fp16 storage of the vocoder's GEMM-only tensors (B200VC_SYNTH_FP16): descriptors only — every ResBlock
    convolution carries fp16 operands, the right mix of fp16 / fp32 outputs, and satisfies the TMA alignment rules."""
    import aicovergen_b200.synth as bs
    from aicovergen_b200.synthetic import make_rvc_checkpoint

    monkeypatch.setattr(bs, "SYNTH_FP16", True)
    m = bs.SynthesizerB200(make_rvc_checkpoint("40k", "v2"), "cpu")
    assert m.half_rb
    pl = bs._Plan(m, 157)
    gemms = [st for st in pl.steps if isinstance(st, tg.TapGemm)]
    half = [op for op in gemms if op.params.dtype & 1]
    assert len(half) == 72 and all(op.name.startswith("rb") for op in half)      # 4 stages x 3 blocks x 3 dilations x 2 convs
    assert all(op.tc_supported() for op in half)
    assert {op.params.dtype for op in half} == {1, 3, 5}    # out fp32 / out fp16 (mid tensor) / out fp32 + fp16 activated copy
    monkeypatch.setattr(bs, "SYNTH_FP16", False)
    m32 = bs.SynthesizerB200(make_rvc_checkpoint("40k", "v2"), "cpu")
    assert not any(st.params.dtype for st in bs._Plan(m32, 157).steps if isinstance(st, tg.TapGemm))
