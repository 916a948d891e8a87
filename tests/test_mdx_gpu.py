"""GPU parity: MDX pass (ConvTDFNet, STFT/iSTFT, chunked process_wave / run_mdx arithmetic) vs the CPU
oracle (oracle/mdx.py; stft/istft/chunking pinned against src/mdx.py)."""
import numpy as np
import pytest
import torch

from aicovergen_b200 import tapgemm as tg
from aicovergen_b200.synthetic import make_mdx_state_dict

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _storage_mode(monkeypatch, request):
    """The U-Net's default storage is fp16 (B200VC_MDX_FP16=1).  Tests on the round-1 RAW random checkpoints pin TF32 storage:
    raw BatchNorm statistics drive activations to 1e5..1e10, beyond fp16's range; fp16 tests use trained-like checkpoints."""
    import aicovergen_b200.mdx as bm
    if "fp16" not in request.node.name:
        monkeypatch.setattr(bm, "MDX_FP16", False)


def rel_rms(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).pow(2).mean().sqrt() / (b.pow(2).mean().sqrt() + 1e-20)).item()


def song(n, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 44100.0
    x = np.stack([0.3 * np.sin(2 * np.pi * 220 * t) + 0.2 * np.sin(2 * np.pi * 554.4 * t + 1.0),
                  0.3 * np.sin(2 * np.pi * 329.6 * t) + 0.2 * np.sin(2 * np.pi * 440 * t + 0.3)])
    x = x * (0.6 + 0.4 * np.sin(2 * np.pi * 0.5 * t)) + 0.05 * rng.standard_normal((2, n))
    return x.astype(np.float32)


@pytest.mark.parametrize("backend,tol", [(tg.BACKEND_SIMT, 3e-5), (tg.BACKEND_TC, 8e-3)])
@pytest.mark.parametrize("cfg", [dict(dim_f=256, dim_t=32, g=8, n=3), dict(dim_f=3072, dim_t=256, g=48, n=5)])
def test_convtdfnet_parity(backend, tol, cfg):
    from aicovergen_b200.mdx import ConvTDFNetB200
    from oracle import mdx as om

    sd = make_mdx_state_dict(**cfg)
    B = 2 if cfg["dim_f"] < 1000 else 1
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 4, cfg["dim_f"], cfg["dim_t"], generator=g) * 3.0
    ref = om.convtdfnet(sd, x)
    net = ConvTDFNetB200(sd, "cuda:0", backend)
    got = torch.from_numpy(net.run(None, {"input": x.numpy()})[0])
    e = rel_rms(got, ref)
    print(f"[mdx net {'tc' if backend else 'simt'} {cfg['dim_f']}x{cfg['dim_t']}] rel rms err {e:.3e} (ref rms {ref.pow(2).mean().sqrt():.3e})")
    assert torch.isfinite(got).all() and e < tol


@pytest.mark.parametrize("dim_f,dim_t,n_fft", [(256, 16, 2048), (3072, 256, 7680), (2048, 256, 5120), (3072, 512, 6144)])
def test_stft_istft_api_parity(dim_f, dim_t, n_fft):
    from aicovergen_b200.mdx import MDXModel
    from oracle import mdx as om

    mp = om.MdxParams(dim_f, dim_t, n_fft)
    m = MDXModel("cuda:0", dim_f, dim_t, n_fft)
    x = torch.from_numpy(song(mp.chunk_size * 2, 3).reshape(2, 2, mp.chunk_size).transpose(1, 0, 2).copy())   # [B=2, 2, chunk]
    ref = mp.stft(x)
    got = m.stft(x.cuda()).cpu()
    e1 = rel_rms(got, ref)
    back_ref = mp.istft(ref)
    back = m.istft(ref.cuda()).cpu()
    e2 = rel_rms(back, back_ref)
    print(f"[mdx stft {dim_f}/{n_fft}] stft rel rms {e1:.3e}; istft rel rms {e2:.3e}")
    assert got.shape == ref.shape and back.shape == back_ref.shape
    assert e1 < 2e-5 and e2 < 2e-5


@pytest.mark.parametrize("backend,tol", [(tg.BACKEND_SIMT, 5e-5), (tg.BACKEND_TC, 8e-3)])
@pytest.mark.parametrize("denoise", [False, True])
def test_run_mdx_arrays_small_geometry(backend, tol, denoise):
    """Whole pass incl. halves / margins / padding / [:-pad] / inverse stem, small geometry so the CPU oracle is quick."""
    from aicovergen_b200.mdx import MDX, MDXModel, run_mdx_arrays
    from oracle import mdx as om

    dim_f, dim_t, n_fft = 256, 16, 2048
    sd = make_mdx_state_dict(dim_f=dim_f, dim_t=dim_t, g=8, n=3)
    wave = song(44100 * 3 + 777, 5)
    mp = om.MdxParams(dim_f, dim_t, n_fft, stem_name="Vocals", compensation=1.035)
    ref_main, ref_inv = om.run_mdx_arrays(wave, mp, lambda s: om.convtdfnet(sd, s), denoise=denoise, m_threads=2)
    model = MDXModel("cuda:0", dim_f, dim_t, n_fft, stem_name="Vocals", compensation=1.035)
    sess = MDX(sd, model, 0, backend=backend)
    main, inv = run_mdx_arrays(sess, wave, denoise=denoise, m_threads=2)
    e1, e2 = rel_rms(main, ref_main), rel_rms(inv, ref_inv)
    a1 = float(np.sqrt(((main - ref_main) ** 2).mean()))
    print(f"[mdx pass {'tc' if backend else 'simt'} denoise={denoise}] main rel {e1:.3e} (abs rms {a1:.3e}), inverse rel {e2:.3e}")
    assert main.shape == ref_main.shape == wave.shape
    assert e1 < tol and e2 < tol


def test_process_wave_full_geometry():
    """Kim_Vocal_2-class geometry (3072 x 256, n_fft 7680): 12 s stereo -> 2 halves x 2 chunks."""
    from aicovergen_b200.mdx import MDX, MDXModel
    from oracle import mdx as om

    dim_f, dim_t, n_fft = 3072, 256, 7680
    sd = make_mdx_state_dict()
    wave = song(44100 * 12, 9)
    wave /= np.abs(wave).max()
    mp = om.MdxParams(dim_f, dim_t, n_fft)
    ref = om.process_wave(wave.copy(), mp, lambda s: om.convtdfnet(sd, s), 2)
    sess = MDX(sd, MDXModel("cuda:0", dim_f, dim_t, n_fft), 0, backend=tg.BACKEND_TC)
    got = sess.process_wave(wave.copy(), 2)
    e = rel_rms(got, ref)
    a = float(np.sqrt(((got - ref) ** 2).mean()))
    print(f"[mdx full geometry tc] rel rms {e:.3e}, abs rms {a:.3e} (ref rms {np.sqrt((ref ** 2).mean()):.3e})")
    assert got.shape == wave.shape and e < 8e-3


def test_first_and_final_conv_row_kernels():
    """The pointwise 4->g / g->4 convolutions at the ends of the U-Net against torch (fp32, same summation order)."""
    from aicovergen_b200 import ops
    g = torch.Generator().manual_seed(2)
    B, T, Fq, ch = 2, 8, 96, 48
    spec = torch.randn(B, 2, T, 2 * Fq, generator=g)
    w4, b4 = torch.randn(ch, 4, generator=g), torch.randn(ch, generator=g)
    x_nchw = spec.view(B, 2, T, Fq, 2).permute(0, 1, 4, 2, 3).reshape(B, 4, T, Fq)            # channel = ch*2 + ri
    ref = torch.relu(torch.einsum("bkth,ck->bthc", x_nchw, w4) + b4)
    out = torch.empty(B, T, Fq, ch, device="cuda")
    ops.mdx_first_conv(spec.cuda(), w4.cuda(), b4.cuda(), out)
    assert (out.cpu() - ref).abs().max() < 1e-5
    wf, bf = torch.randn(4, ch, generator=g) / ch ** 0.5, torch.randn(4, generator=g)
    y = torch.einsum("bthc,kc->bkth", ref, wf) + bf[None, :, None, None]                        # [B,4,T,F]
    ref_spec = y.view(B, 2, 2, T, Fq).permute(0, 1, 3, 4, 2).reshape(B, 2, T, 2 * Fq)
    so = torch.empty(B, 2, T, 2 * Fq, device="cuda")
    ops.mdx_final_conv(out, wf.cuda(), bf.cuda(), so)
    assert (so.cpu() - ref_spec).abs().max() < 1e-4


@pytest.mark.parametrize("cfg", [dict(dim_f=256, dim_t=32, g=8, n=3), dict(dim_f=3072, dim_t=256, g=48, n=5)])
def test_convtdfnet_parity_fp16_storage(cfg, monkeypatch):
    """The U-Net with fp16 activation / weight storage (wgmma f16, fp32 accumulate) — the DEFAULT mode — on
    trained-like checkpoints: same mantissa width as the TF32 path, half the bytes."""
    import aicovergen_b200.mdx as bm
    from oracle import mdx as om

    from aicovergen_b200.synthetic import make_mdx_trained_like
    monkeypatch.setattr(bm, "MDX_FP16", True)
    # trained-like BatchNorm statistics: raw random statistics overflow fp16 at the full geometry (DESIGN.md)
    sd = make_mdx_trained_like(cfg["dim_f"], cfg["dim_t"], {256: 2048, 3072: 7680}[cfg["dim_f"]], g=cfg["g"], n=cfg["n"])
    B = 2 if cfg["dim_f"] < 1000 else 1
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 4, cfg["dim_f"], cfg["dim_t"], generator=g) * 3.0
    ref = om.convtdfnet(sd, x)
    net = bm.ConvTDFNetB200(sd, "cuda:0", tg.BACKEND_TC)
    assert net.half
    got = torch.from_numpy(net.run(None, {"input": x.numpy()})[0])
    e = rel_rms(got, ref)
    print(f"[mdx net fp16 storage {cfg['dim_f']}x{cfg['dim_t']}] rel rms err {e:.3e}")
    assert torch.isfinite(got).all() and e < 3e-3


def test_process_wave_full_geometry_fp16_abs_rms():
    """Kim_Vocal_2-class geometry, default fp16 storage, trained-like checkpoint: 12 s stereo -> 2 halves x 2 chunks;
    the stem is compared in ABSOLUTE RMS on [-1, 1] audio (north_star bar 1e-3)."""
    import aicovergen_b200.mdx as bm
    from aicovergen_b200.synthetic import make_mdx_trained_like
    from oracle import mdx as om

    assert bm.MDX_FP16, "fp16 storage is the default"
    dim_f, dim_t, n_fft = 3072, 256, 7680
    sd = make_mdx_trained_like(dim_f, dim_t, n_fft)
    wave = song(44100 * 12, 9)
    wave /= np.abs(wave).max()
    mp = om.MdxParams(dim_f, dim_t, n_fft)
    ref = om.process_wave(wave.copy(), mp, lambda s: om.convtdfnet(sd, s), 2)
    sess = bm.MDX(sd, bm.MDXModel("cuda:0", dim_f, dim_t, n_fft), 0, backend=tg.BACKEND_TC)
    assert sess.ort.half
    got = sess.process_wave(wave.copy(), 2)
    a = float(np.sqrt(((got - ref) ** 2).mean()))
    r = float(np.sqrt((ref ** 2).mean()))
    print(f"[mdx full geometry fp16] abs rms err {a:.3e} (ref rms {r:.3e}, rel {a / r:.2e})")
    assert got.shape == wave.shape and r > 1e-2 and a < 1e-3 and a / r < 5e-3
