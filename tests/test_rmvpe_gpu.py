"""GPU parity: RMVPE (infer_from_audio plug point) vs the CPU oracle restatement (oracle/rmvpe.py,
pinned against src/rmvpe.py).  BASELINE.json config 1: 10 s 100->1000 Hz sine sweep at 16 kHz."""
import numpy as np
import pytest
import torch

from aicovergen_b200 import tapgemm as tg
from aicovergen_b200.synthetic import make_rmvpe_state_dict

pytestmark = pytest.mark.gpu


def sweep(seconds):
    t = np.arange(int(16000 * seconds)) / 16000.0
    return (0.5 * np.sin(2 * np.pi * (100 * t + 45 * t * t))).astype(np.float32)


@pytest.mark.parametrize("weights", ["trained_like", "raw"])
@pytest.mark.parametrize("seconds", [2.93, 10.0])
def test_rmvpe_f0_parity(seconds, weights):
    """BASELINE.json config 1 (10 s sweep) through the `infer_from_audio` plug point: coarse pitch indices bit-exact.

    Salience tolerance: a pure sine sweep leaves most mel bins at leakage level, right around the 1e-5 clamp of the
    log (rmvpe.py:324).  There the fp32 STFT's own rounding (~1e-6 absolute, whether FFT as in torch or DFT-GEMM as here)
    is a percent-level relative error, i.e. ~1e-2 in log-mel; pushed through the network that is 4e-5 .. 1e-3 of salience
    (reproduced on the CPU alone by swapping torch.stft for a direct fp32 DFT in the oracle).  The reference's own CPU and
    CUDA paths differ by the same amount.  The network itself is held to 5e-5 on an identical log-mel input in
    test_rmvpe_net_parity_given_logmel below; broadband inputs are at 1e-5 end to end."""
    from aicovergen_b200.rmvpe import RMVPEB200
    from aicovergen_b200.synthetic import make_rmvpe_trained_like
    from oracle import rmvpe as orm

    sd = make_rmvpe_trained_like() if weights == "trained_like" else make_rmvpe_state_dict()
    x = sweep(seconds)
    a = torch.from_numpy(x)[None]
    hid_ref = orm.mel2hidden(sd, orm.log_mel(a))[0]
    f0_ref = orm.decode(hid_ref.numpy().copy(), 0.03)
    pitch_ref, pitchf_ref = orm.coarse_pitch(f0_ref, 0)

    # trained-like weights: the default backend (U-Net on the tensor cores, 3xTF32 split operands); round-1 raw weights: the exact-fp32
    # SIMT kernel (their unstructured salience head turns any rounding difference into a different octave)
    net = RMVPEB200(sd, device="cuda:0", backend=tg.BACKEND_TC if weights == "trained_like" else tg.BACKEND_SIMT)
    sal = net.salience_from_audio(torch.from_numpy(x).cuda()).cpu()
    err = (sal - hid_ref).abs().max().item()
    print(f"[rmvpe {weights} {seconds}s] salience max abs err {err:.3e} over {tuple(sal.shape)}")
    f0 = net.infer_from_audio(x, thred=0.03)
    assert f0.shape == f0_ref.shape == (1 + len(x) // 160,)
    pitch, pitchf = orm.coarse_pitch(f0, 0)
    # A frame whose reference F0 lies within 1e-6 relative of a rounding boundary of the quantiser is a tie at float32
    # resolution (one float32 ulp is ~6e-8 relative; the salience it is decoded from is float32 and carries the tolerance
    # asserted below): no fp32 implementation can place it reliably, so there either neighbouring index is accepted.
    # The 10 s sweep has one such frame (74: 4.3e-8 relative from the boundary); every other frame must match exactly.
    up, dn = orm.coarse_pitch(f0_ref * (1 + 1e-6), 0)[0], orm.coarse_pitch(f0_ref * (1 - 1e-6), 0)[0]
    tie = up != dn
    mism = int(((pitch != pitch_ref) & ~tie).sum())
    both = (f0 > 0) & (f0_ref > 0)
    rel = np.abs(f0 - f0_ref)[both] / f0_ref[both]
    print(f"[rmvpe {weights} {seconds}s] coarse-pitch mismatches {mism}/{len(pitch)} (+ {int((pitch != pitch_ref)[tie].sum())} of "
          f"{int(tie.sum())} float32 ties); f0 max rel diff {rel.max():.3e}; voiced {(f0_ref > 0).mean():.2f}; "
          f"{len(np.unique(pitch_ref))} distinct levels")
    assert err < (1.5e-3 if weights == "trained_like" else 3e-4)
    assert mism == 0, "coarse pitch indices must match the reference bit for bit"
    assert ((pitch == up) | (pitch == dn))[tie].all(), "a tie frame must take one of the two indices it lies between"
    assert np.array_equal(f0 > 0, f0_ref > 0) and rel.max() < 1e-3


@pytest.mark.parametrize("backend,bar", [(tg.BACKEND_TC, 5e-5), (tg.BACKEND_SIMT, 2e-5)])
@pytest.mark.parametrize("kind", ["sweep", "vocal"])
def test_rmvpe_net_parity_given_logmel(kind, backend, bar):
    """`RMVPE.mel2hidden(mel)` plug point (rmvpe.py:350-357): U-Net + BiGRU + head on the ORACLE's log-mel, i.e. without the
    STFT front-end in the comparison — the network's own error against the fp32 CPU oracle."""
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from siggen import vocal_like
    from aicovergen_b200.rmvpe import RMVPEB200
    from aicovergen_b200.synthetic import make_rmvpe_trained_like
    from oracle import rmvpe as orm

    sd = make_rmvpe_trained_like()
    x = sweep(4.0) if kind == "sweep" else vocal_like(4.0, seed=9)
    mel = orm.log_mel(torch.from_numpy(x)[None])
    ref = orm.mel2hidden(sd, mel)[0]
    net = RMVPEB200(sd, device="cuda:0", backend=backend)
    got = net.mel2hidden(mel.cuda())[0].cpu()
    err = (got - ref).abs().max().item()
    f0, f0_ref = net.decode(got.numpy()), orm.decode(ref.numpy().copy(), 0.03)
    mism = int((orm.coarse_pitch(f0)[0] != orm.coarse_pitch(f0_ref)[0]).sum())
    print(f"[rmvpe net {'3xTF32 wgmma' if backend == tg.BACKEND_TC else 'fp32 simt'} | oracle log-mel, {kind}] salience max abs err {err:.3e}; "
          f"coarse-pitch mismatches {mism}/{len(f0)}")
    assert got.shape == ref.shape and err < bar and mism == 0
    # the front-end alone: device log-mel vs torch.stft log-mel on bins above the clamp region
    pl = net._plan(len(x))
    net.salience_from_audio(torch.from_numpy(x).cuda())
    lm = torch.log(torch.clamp(pl.melp[:pl.n_frames].cpu(), min=1e-5)).t()
    hi = mel[0] > np.log(1e-3)
    e_hi = (lm - mel[0])[hi].abs().max().item()
    print(f"[rmvpe front-end, {kind}] log-mel max abs err {e_hi:.3e} on {int(hi.sum())} bins above 1e-3, {(lm - mel[0]).abs().max().item():.3e} on all")
    assert e_hi < 2e-3


def test_rmvpe_decode_kernel_exact():
    """The decode kernel alone reproduces numpy's float32/float64 summation order bit for bit."""
    from aicovergen_b200 import ops
    from oracle import rmvpe as orm

    g = torch.Generator().manual_seed(3)
    sal = torch.rand(2000, 360, generator=g)
    sal[5] = 0.01                      # below threshold
    sal[6, :] = 0.5                    # full tie -> first index
    sal[7, 359] = 2.0                  # edge window
    sal[8, 0] = 2.0
    ref = orm.decode(sal.numpy().copy(), 0.03)
    f0 = torch.empty(2000, dtype=torch.float64, device="cuda")
    cents = torch.empty(2000, dtype=torch.float64, device="cuda")
    ops.rmvpe_decode(sal.cuda(), f0, 2000, 0.03, cents=cents)
    got = f0.cpu().numpy()
    ulp = np.abs(got - ref) / np.maximum(np.abs(ref), 1e-300)
    print(f"[rmvpe decode] device f0 max rel diff {ulp.max():.3e}, exact {(got == ref).mean():.4f}")
    assert ulp.max() < 1e-14
    # host finish (what infer_from_audio does) must be bit-identical to numpy
    c = cents.cpu().numpy()
    f0h = 10 * (2 ** (c / 1200))
    f0h[f0h == 10] = 0
    print(f"[rmvpe decode] host-finished f0 exact {(f0h == ref).mean():.4f}")
    assert np.array_equal(f0h, ref)
    assert (orm.coarse_pitch(got)[0] == orm.coarse_pitch(ref)[0]).all()


@pytest.mark.parametrize("ver", ["1", "2", "3"])
@pytest.mark.parametrize("T", [37, 1024, 24608])
def test_bigru_kernel_matches_torch_gru(T, ver, monkeypatch):
    """b200vc_bigru (2 clusters x 8 CTAs, one DSMEM hop per step) against torch.nn.GRU(384, 256, bidirectional) on the CPU:
    24 608 steps = the F0 of a 4-min song."""
    from aicovergen_b200 import ops

    monkeypatch.setenv("B200VC_GRU", ver)       # 1: cluster barrier per step (default); 2: st.async per value; 3: bulk copy per peer
    g = torch.Generator().manual_seed(T)
    gru = torch.nn.GRU(384, 256, num_layers=1, batch_first=True, bidirectional=True).eval()
    x = torch.randn(1, T, 384, generator=g)
    with torch.no_grad():
        ref = gru(x)[0][0]
        xp = torch.cat([x[0] @ gru.weight_ih_l0.t() + gru.bias_ih_l0, x[0] @ gru.weight_ih_l0_reverse.t() + gru.bias_ih_l0_reverse], 1)
    whh = torch.stack([gru.weight_hh_l0, gru.weight_hh_l0_reverse]).detach().contiguous().cuda()
    bhh = torch.stack([gru.bias_hh_l0, gru.bias_hh_l0_reverse]).detach().contiguous().cuda()
    out = torch.empty(T, 512, device="cuda")
    ops.bigru(xp.contiguous().cuda(), whh, bhh, out, 256)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    ops.bigru(xp.contiguous().cuda(), whh, bhh, out, 256)
    e.record()
    torch.cuda.synchronize()
    err = (out.cpu() - ref).abs().max().item()
    print(f"[bigru v{ver} T={T}] max abs err {err:.3e}; {s.elapsed_time(e):.2f} ms = {s.elapsed_time(e) * 1e3 / T:.3f} us/step")
    assert err < 2e-5
