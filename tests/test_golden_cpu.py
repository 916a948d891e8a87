"""The oracle restatements reproduce the golden vectors generated from the UNMODIFIED reference
(tools/make_golden.py) — runs anywhere, no GPU, no reference checkout."""
import os

import numpy as np
import torch

from siggen import stereo_tones, vocal_like

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_synth_oracle_vs_golden():
    from aicovergen_b200.synthetic import make_rvc_checkpoint
    from oracle import synth as osyn

    z = np.load(os.path.join(G, "synth_v2_40k.npz"))
    cpt = make_rvc_checkpoint("40k", "v2", seed=int(z["ckpt_seed"]))
    P = z["phone"].shape[1]
    nz, ns = osyn.draw_noise(int(z["noise_seed"]), P, 192, 400)
    o, lat = osyn.infer(cpt, torch.from_numpy(z["phone"]), torch.from_numpy(z["pitch"]), torch.from_numpy(z["pitchf"]),
                        torch.tensor([0]), nz, ns, return_all=True)
    assert np.abs(o.numpy()[0, 0] - z["out"]).max() < 5e-6
    assert np.abs(lat["m_p"].numpy() - z["m_p"]).max() < 1e-5


def test_rmvpe_oracle_vs_golden():
    from aicovergen_b200.synthetic import make_rmvpe_state_dict
    from oracle import rmvpe as orm

    z = np.load(os.path.join(G, "rmvpe.npz"))
    sd = make_rmvpe_state_dict(seed=int(z["ckpt_seed"]))
    x = vocal_like(float(z["seconds"]), seed=int(z["audio_seed"]))
    f0 = orm.infer_from_audio(sd, x, 0.03)
    assert f0.shape == z["f0"].shape
    assert np.array_equal(orm.coarse_pitch(f0)[0], orm.coarse_pitch(z["f0"])[0])
    assert np.abs(f0 - z["f0"]).max() / z["f0"].max() < 1e-5


def test_pipeline_oracle_vs_golden():
    from aicovergen_b200.synthetic import make_hubert_state_dict, make_rmvpe_state_dict, make_rvc_checkpoint
    from oracle import pipeline as opipe

    z = np.load(os.path.join(G, "vc_pipeline.npz"))
    audio = vocal_like(float(z["seconds"]), seed=int(z["audio_seed"]))
    xs = {k: int(z[k]) for k in ("x_pad", "x_query", "x_center", "x_max")}
    out, info = opipe.pipeline(make_hubert_state_dict(seed=777), make_rvc_checkpoint("40k", "v2", seed=1234),
                               make_rmvpe_state_dict(seed=4321), audio, index=None, seed=int(z["noise_seed"]),
                               return_all=True, **xs)
    assert len(info["opt_ts"]) >= 1
    d = np.abs(out.astype(np.int32) - z["out_int16"].astype(np.int32))
    assert out.shape == z["out_int16"].shape and d.max() <= 12 and np.sqrt((d.astype(float) ** 2).mean()) < 1.5


def test_mdx_oracle_vs_golden():
    from aicovergen_b200.synthetic import make_mdx_state_dict
    from oracle import mdx as om

    z = np.load(os.path.join(G, "mdx_small.npz"))
    dim_f, dim_t, n_fft = int(z["dim_f"]), int(z["dim_t"]), int(z["n_fft"])
    sd = make_mdx_state_dict(dim_f=dim_f, dim_t=dim_t, g=8, n=3, seed=int(z["ckpt_seed"]))
    mp = om.MdxParams(dim_f, dim_t, n_fft)
    wave = stereo_tones(int(z["n"]), seed=int(z["wave_seed"]))
    got = om.process_wave(wave.copy(), mp, lambda s: om.convtdfnet(sd, s), 2)
    assert got.shape == z["processed"].shape
    assert np.abs(got - z["processed"]).max() < 1e-6
    spec = mp.stft(torch.from_numpy(wave[:, :mp.chunk_size].copy())[None])
    assert np.allclose(spec[0, :, :8, :4].numpy(), z["spec_slice"], rtol=0, atol=1e-6)
