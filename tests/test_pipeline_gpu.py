"""GPU parity of the whole RVC path: VC.pipeline (GPU operators) vs oracle/pipeline.py (pinned against the
reference's unmodified VC.pipeline).  Bar (BASELINE.json north_star): coarse F0 indices bit-exact, fp32 waveform
within 1e-3 RMS."""
import os
import sys
import tempfile
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from aicovergen_b200.synthetic import (make_hubert_state_dict, make_ivf_index_data, make_rmvpe_state_dict,  # noqa: E402
                                       make_rvc_checkpoint)

pytestmark = pytest.mark.gpu


def vocal_like(seconds, sr=16000, seed=7):
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    t = np.arange(n) / sr
    f0 = 220.0 * 2 ** (0.5 * np.sin(2 * np.pi * 0.2 * t)) * 2 ** (30 / 1200 * np.sin(2 * np.pi * 5.5 * t))
    phase = 2 * np.pi * np.cumsum(f0) / sr
    x = sum(np.sin(k * phase) / k for k in range(1, 9))
    burst = ((t % 3.0) > 2.6)
    x = np.where(burst, rng.standard_normal(n) * 0.7, x)
    x = x + 0.1 * rng.standard_normal(n)
    x = x * np.where((t % 1.7) > 1.62, 0.02, 1.0)
    return (0.5 * x / np.abs(x).max()).astype(np.float32)


@pytest.mark.parametrize("with_index", [False, "npz", "faiss"])
def test_vc_pipeline_parity(with_index):
    from aicovergen_b200.hubert import HubertB200
    from aicovergen_b200.index import write_index_npz
    from aicovergen_b200.rmvpe import RMVPEB200
    from aicovergen_b200.synth import SynthesizerB200
    from aicovergen_b200.vc_infer_pipeline import VC
    from oracle import hubert as ohub
    from oracle import pipeline as opipe
    from oracle.index import IvfFlatIndex

    hsd, rsd, cpt = make_hubert_state_dict(), make_rmvpe_state_dict(), make_rvc_checkpoint("40k", "v2")
    audio = vocal_like(7.7)
    xs = dict(x_pad=1, x_query=1, x_center=3, x_max=4)        # small constants so 7.7 s already needs 2 cuts
    index, file_index = None, ""
    if with_index:
        base = ohub.extract_features(hsd, torch.from_numpy(vocal_like(4.0, seed=3))[None], 12)[0]
        cent, vecs = make_ivf_index_data(base, n_total=4000, nlist=64)
        index = IvfFlatIndex(cent, vecs)
        if with_index == "npz":
            tmp = tempfile.NamedTemporaryFile(suffix=".npz", delete=False)
            tmp.close()
            write_index_npz(tmp.name, cent, vecs)
        else:   # the binary IndexIVFFlat layout faiss writes (what RVC voice models ship): read back through faiss_io
            from aicovergen_b200.faiss_io import write_ivfflat
            tmp = tempfile.NamedTemporaryFile(suffix="_IVF64_Flat_nprobe_1.index", delete=False)
            tmp.close()
            write_ivfflat(tmp.name, cent, vecs, index.assign)
        file_index = tmp.name
    ref_i16, info = opipe.pipeline(hsd, cpt, rsd, audio.copy(), index=index, seed=5, return_all=True, **xs)

    cfg = types.SimpleNamespace(device="cuda:0", is_half=True, **xs)
    vc = VC(40000, cfg)
    vc.model_rmvpe = RMVPEB200(rsd, device="cuda:0")
    vc.set_noise_seed(5)
    vc.keep_float = True
    hubert = HubertB200(hsd, "cuda:0")
    net_g = SynthesizerB200(cpt, "cuda:0")
    times = [0, 0, 0]
    out = vc.pipeline(hubert, net_g, 0, audio.copy(), "x.wav", times, 0, "rmvpe", file_index, 0.5, 1, 3, 40000, 0, 0.25,
                      "v2", 0.33, 128)
    if with_index:
        os.unlink(file_index)
    assert out.dtype == np.int16 and out.shape == ref_i16.shape
    assert len(info["opt_ts"]) >= 1
    # F0 indices: recompute through the same get_f0 the pipeline used
    from scipy import signal
    pad = np.pad(signal.filtfilt(opipe.bh, opipe.ah, audio), (16000 * xs['x_pad'], 16000 * xs['x_pad']), mode="reflect")
    pitch, pitchf = vc.get_f0("x.wav", pad, len(pad) // 160, 0, "rmvpe", 3, 128)
    p_len = len(pad) // 160
    mism = int((pitch[:p_len] != info["pitch"]).sum())
    e_float = float(np.sqrt(((vc.last_float_output.astype(np.float64) - info["float_out"]) ** 2).mean()))
    ref_rms = float(np.sqrt((info["float_out"].astype(np.float64) ** 2).mean()))
    d16 = np.abs(out.astype(np.int32) - ref_i16.astype(np.int32))
    print(f"[pipeline index={with_index}] coarse-pitch mismatches {mism}/{p_len}; float waveform abs rms err {e_float:.3e} "
          f"(ref rms {ref_rms:.3e}); int16 max diff {d16.max()} rms {np.sqrt((d16.astype(float) ** 2).mean()):.2f}; cuts {info['opt_ts']}")
    assert mism == 0
    assert e_float < 1e-3
    # the F0-on-a-side-stream schedule (rmvpe overlapped with the HuBERT / index half of the segments) computes the same
    # numbers in a different order: bit-identical utterance, three times in a row (eager, recorded plans, graph replays)
    import aicovergen_b200.vc_infer_pipeline as vcmod
    if with_index != "npz":
        return
    prev = vcmod.F0_OVERLAP
    try:
        outs = []
        for flag in (False, True, True, True):
            vcmod.F0_OVERLAP = flag
            vc.set_noise_seed(5)
            outs.append(vc.pipeline(hubert, net_g, 0, audio.copy(), "x.wav", times, 0, "rmvpe", "", 0.5, 1, 3, 40000, 0, 0.25,
                                    "v2", 0.33, 128))
    finally:
        vcmod.F0_OVERLAP = prev
    assert all(np.array_equal(outs[0], o) for o in outs[1:])


def test_device_filtfilt_matches_scipy():
    """Device zero-phase HPF (sos cascade, block-parallel) vs scipy: ~1e-12 to sosfiltfilt, and within the reference's own
    numerical noise (ba-form filtfilt vs sosfiltfilt differ by ~7e-7) of the exact call at vc_infer_pipeline.py:513."""
    from scipy import signal

    from aicovergen_b200 import ops
    from aicovergen_b200.vc_infer_pipeline import ah, bh

    x = vocal_like(23.0, seed=2)
    ref_ba = signal.filtfilt(bh, ah, x)
    ref_sos = signal.sosfiltfilt(signal.tf2sos(bh, ah), x, padtype="odd", padlen=18)
    got = ops.filtfilt(torch.from_numpy(x).cuda(), bh, ah).cpu().numpy()
    e_sos, e_ba = np.abs(got - ref_sos).max(), np.abs(got - ref_ba).max()
    print(f"[filtfilt] max abs diff vs scipy.sosfiltfilt {e_sos:.2e}, vs scipy.filtfilt(ba) {e_ba:.2e} (scipy ba vs sos {np.abs(ref_ba - ref_sos).max():.2e})")
    assert e_sos < 1e-10 and e_ba < 5e-6


def test_device_change_rms_and_int16_match_host():
    from aicovergen_b200 import ops
    from oracle import pipeline as opipe

    rng = np.random.default_rng(3)
    a = vocal_like(6.3, seed=4).astype(np.float64) * 0.8
    out = (0.4 * rng.standard_normal(int(6.3 * 40000))).astype(np.float32) * (0.5 + 0.5 * np.sin(np.arange(int(6.3 * 40000)) / 9000.0)).astype(np.float32)
    ref = opipe.change_rms(a.copy(), 16000, out.copy(), 40000, 0.25)
    d = torch.from_numpy(out.copy()).cuda()
    ops.change_rms(torch.from_numpy(a).cuda(), 16000, d, 40000, 0.25)
    got = d.cpu().numpy()
    rel = np.abs(got - ref).max() / np.abs(ref).max()
    print(f"[change_rms] max rel diff {rel:.2e}")
    assert rel < 2e-5
    for scale in (1.0, 3.7):          # second case triggers the peak guard
        x = (ref * scale).astype(np.float32)
        audio_max = np.abs(x).max() / 0.99
        m = 32768 / audio_max if audio_max > 1 else 32768
        want = (x * m).astype(np.int16)
        have = ops.to_int16_peak_guard(torch.from_numpy(x).cuda()).cpu().numpy()
        assert np.abs(have.astype(np.int32) - want.astype(np.int32)).max() <= 1
