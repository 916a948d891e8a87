"""GPU parity: synthesizer (net_g.infer plug point) vs the CPU oracle restatement
(oracle/synth.py, pinned against infer_pack/models.py) on seeded synthetic weights."""
import pytest
import torch

from aicovergen_b200 import tapgemm as tg
from aicovergen_b200.synthetic import make_rvc_checkpoint

pytestmark = pytest.mark.gpu


def rms(x):
    return x.double().pow(2).mean().sqrt().item()


def _inputs(P, seed, in_dim=768):
    g = torch.Generator().manual_seed(seed)
    phone = torch.randn(1, P, in_dim, generator=g)
    pitchf = 220.0 * 2 ** (0.5 * torch.sin(torch.arange(P) * 0.05)) + torch.randn(P, generator=g)
    pitchf[P // 5: P // 5 + 12] = 0.0
    pitchf = pitchf[None].float()
    pitch = torch.randint(1, 255, (1, P), generator=g)
    return phone, pitch, pitchf


@pytest.mark.parametrize("backend,tol_wave,tol_lat", [(tg.BACKEND_SIMT, 2e-5, 2e-5), (tg.BACKEND_TC, 1e-3, 3e-3)])
@pytest.mark.parametrize("P", [157, 700])
def test_synth_infer_parity(backend, tol_wave, tol_lat, P):
    from aicovergen_b200.synth import SynthesizerB200
    from oracle import synth as osynth

    cpt = make_rvc_checkpoint("40k", "v2", seed=1234)
    phone, pitch, pitchf = _inputs(P, P)
    sid = torch.tensor([0])
    nz, ns = osynth.draw_noise(7, P, 192, 400)
    ref, lat = osynth.infer(cpt, phone, pitch, pitchf, sid, nz, ns, return_all=True)

    net = SynthesizerB200(cpt, "cuda:0", backend=backend)
    o, _, (z, z_p, m_p, logs_p) = net.infer(phone.cuda(), torch.tensor([P]).cuda(), pitch.cuda(), pitchf.cuda(),
                                            sid.cuda(), noise_z=nz.cuda(), noise_src=ns.cuda())
    torch.cuda.synchronize()
    name = "tc" if backend == tg.BACKEND_TC else "simt"
    errs = {}
    for k, got in (("m_p", m_p), ("logs_p", logs_p), ("z_p", z_p), ("z", z)):
        errs[k] = rms(got.cpu() - lat[k]) / rms(lat[k])
        print(f"[synth {name} P={P}] {k}: rel rms err {errs[k]:.3e}")
    e_abs = rms(o.cpu() - ref)
    print(f"[synth {name} P={P}] waveform: abs rms err {e_abs:.3e} (ref rms {rms(ref):.3e}, rel {e_abs / rms(ref):.3e})")
    assert torch.isfinite(o).all()
    for k, e in errs.items():
        assert e < tol_lat, (k, e)
    assert e_abs < tol_wave, e_abs
    # second call with the same plan must be deterministic
    o2 = net.infer(phone.cuda(), torch.tensor([P]).cuda(), pitch.cuda(), pitchf.cuda(), sid.cuda(),
                   noise_z=nz.cuda(), noise_src=ns.cuda())[0]
    torch.cuda.synchronize()
    assert torch.equal(o, o2)


@pytest.mark.parametrize("C,K,stride,pad", [(256, 80, 40, 20), (64, 4, 2, 1), (32, 1, 1, 0), (512, 10, 5, 0)])
def test_conv1d_from1_row_kernel(C, K, stride, pad):
    """NSF noise_convs / HuBERT conv0 as a row kernel: out = res + bias + Conv1d(1, C, K, stride, padding)(src)."""
    import torch.nn.functional as F

    from aicovergen_b200 import ops
    from aicovergen_b200 import tapgemm as tg
    g = torch.Generator().manual_seed(C + K)
    n = 4000
    src = torch.randn(n, generator=g)
    w, b = torch.randn(C, K, generator=g) / K ** 0.5, torch.randn(C, generator=g)
    ref = F.conv1d(src[None, None], w[:, None, :], b, stride=stride, padding=pad)[0].t().contiguous()     # [T, C]
    T = ref.shape[0]
    res = torch.randn(T, C, generator=g)
    out = res.clone().cuda()
    out2 = torch.empty(T, C, device="cuda")
    ops.conv1d_from1(src.cuda(), w.cuda(), out, stride, -pad, bias=b.cuda(), res=out, out2=out2, act2=tg.ACT_LRELU, act2_p=0.1)
    torch.cuda.synchronize()
    want = ref + res
    assert (out.cpu() - want).abs().max() < 1e-4
    assert (out2.cpu() - F.leaky_relu(want, 0.1)).abs().max() < 1e-4


def test_synth_infer_parity_fp16_resblocks(monkeypatch):
    """Same parity bar as the TF32 path (waveform abs RMS <= 1e-3) with the ResBlock operands stored in fp16."""
    import aicovergen_b200.synth as bs
    from oracle import synth as osynth

    monkeypatch.setattr(bs, "SYNTH_FP16", True)
    P = 157
    cpt = make_rvc_checkpoint("40k", "v2", seed=1234)
    phone, pitch, pitchf = _inputs(P, P)
    sid = torch.tensor([0])
    nz, ns = osynth.draw_noise(7, P, 192, 400)
    ref = osynth.infer(cpt, phone, pitch, pitchf, sid, nz, ns)
    net = bs.SynthesizerB200(cpt, "cuda:0")
    assert net.half_rb
    o = net.infer(phone.cuda(), torch.tensor([P]).cuda(), pitch.cuda(), pitchf.cuda(), sid.cuda(),
                  noise_z=nz.cuda(), noise_src=ns.cuda())[0]
    torch.cuda.synchronize()
    e_abs = rms(o.cpu() - ref)
    print(f"[synth fp16 resblocks P={P}] waveform: abs rms err {e_abs:.3e} (ref rms {rms(ref):.3e})")
    assert torch.isfinite(o).all() and e_abs < 1e-3, e_abs
