"""Pins the oracle restatements against what the UNMODIFIED reference code computes on the same seeded inputs.  The
reference outputs are stored in tests/golden/oracle_pins.npz (tools/make_golden.py pins): bit-exact comparisons as the
SHA-256 of the reference tensor, tolerance comparisons on a fixed seeded sample of output positions."""
import hashlib
import os

import numpy as np
import pytest
import torch

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def pins():
    return np.load(os.path.join(G, "oracle_pins.npz"))


def _sha(t):
    a = t.numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_synth_oracle_matches_reference(pins):
    from aicovergen_b200.synthetic import make_rvc_checkpoint
    from oracle import synth as osyn

    cpt = make_rvc_checkpoint("40k", "v2")
    P = 48
    g = torch.Generator().manual_seed(1)
    phone = torch.randn(1, P, 768, generator=g)
    pitch = torch.randint(1, 255, (1, P), generator=g)
    pitchf = torch.rand(1, P, generator=g) * 300 + 80
    pitchf[:, 7:15] = 0
    nz, ns = osyn.draw_noise(11, P, 192, 400)
    o = osyn.infer(cpt, phone, pitch, pitchf, torch.tensor([0]), nz, ns).numpy().ravel()
    assert o.size == int(pins["synth_n"])
    assert np.abs(o[pins["synth_idx"]] - pins["synth_out"]).max() < 2e-6


def test_synthetic_checkpoints_load_strictly_in_reference(pins):
    """Every parameter the reference modules declare (name and shape) is in the synthetic checkpoints, and nothing else."""
    from aicovergen_b200.synthetic import make_rmvpe_state_dict, make_rvc_checkpoint

    def names(sd):
        return sorted(f"{k}:{tuple(v.shape)}" for k, v in sd.items())

    for key, up in (("40k", 400), ("48k_v2", 480), ("32k", 320)):
        cpt = make_rvc_checkpoint(key, "v2")
        assert names(cpt["weight"]) == list(pins[f"params_{key}"]), key
        assert int(np.prod(cpt["config"][12])) == up
    assert names(make_rmvpe_state_dict()) == list(pins["params_rmvpe"])


def test_rmvpe_oracle_matches_reference(pins):
    from aicovergen_b200.synthetic import make_rmvpe_state_dict
    from oracle import rmvpe as orm
    from siggen import vocal_like

    sd = make_rmvpe_state_dict()
    x = vocal_like(2.5)
    f_ref = pins["rmvpe_f0"]
    f_or = orm.infer_from_audio(sd, x, 0.03)
    assert f_ref.shape == f_or.shape
    assert np.abs(f_ref - f_or).max() / f_ref.max() < 1e-5
    assert _sha(orm.log_mel(torch.from_numpy(x)[None])) == str(pins["rmvpe_mel_sha"])
    # decode restatement is bit-exact given the same salience
    h = pins["rmvpe_salience"]
    assert np.array_equal(orm.decode(h.copy(), 0.03), pins["rmvpe_decode"])


@pytest.mark.parametrize("with_index", [False, True])
def test_pipeline_oracle_matches_reference(pins, with_index):
    """Whole VC.pipeline: 2 segments (small x_* so it stays cheap), rmvpe F0, protect + RMS mix (+ index)."""
    from aicovergen_b200.synthetic import (make_hubert_state_dict, make_ivf_index_data, make_rmvpe_state_dict,
                                           make_rvc_checkpoint)
    from oracle import hubert as ohub
    from oracle import pipeline as opipe
    from oracle.index import IvfFlatIndex
    from siggen import vocal_like

    hsd = make_hubert_state_dict(layers=2)
    cpt = make_rvc_checkpoint("40k", "v2")
    rsd = make_rmvpe_state_dict()
    audio = vocal_like(5.3)
    xs = dict(x_pad=1, x_query=1, x_center=2, x_max=3)
    index = None
    if with_index:
        base = ohub.extract_features(hsd, torch.from_numpy(vocal_like(3.0, seed=3))[None], 2)[0]
        cent, vecs = make_ivf_index_data(base, n_total=2000, nlist=40)
        index = IvfFlatIndex(cent, vecs)
    # the same 2-layer hubert the reference run used: temporarily patch the layer count
    orig = ohub.extract_features
    ohub.extract_features = lambda sd, src, layer=12, n_heads=12: orig(sd, src, 2, n_heads)
    try:
        out, info = opipe.pipeline(hsd, cpt, rsd, audio.copy(), index=index, seed=5, return_all=True, **xs)
    finally:
        ohub.extract_features = orig
    k = f"pipeline_{int(with_index)}"
    assert len(info["opt_ts"]) >= 1, "test must exercise the cut-point path"
    assert out.size == int(pins[k + "_n"]) and out.dtype == np.int16
    diff = np.abs(out[pins[k + "_idx"]].astype(np.int32) - pins[k + "_out"].astype(np.int32))
    # the only arithmetic difference is fp32 reassociation in the GRU restatement (f0 differs ~1e-6 relative,
    # which the random-weight synthesizer amplifies to ~1e-4 on the waveform)
    assert diff.max() <= 12, diff.max()
    assert np.sqrt((diff.astype(np.float64) ** 2).mean()) < 1.5


def test_mdx_oracle_matches_reference(pins):
    """mdx.py's own MDXModel.stft/istft and MDX.process_wave (2 threads, margins, padding) with a fake ORT
    session running the restated net, vs oracle/mdx.py."""
    from aicovergen_b200.synthetic import make_mdx_state_dict
    from oracle import mdx as om

    dim_f, dim_t, n_fft = 256, 16, 2048         # small geometry: chunk = 1024*15 samples, trim 1024
    sd = make_mdx_state_dict(dim_f=dim_f, dim_t=dim_t, g=8, n=3)
    net = lambda spec: om.convtdfnet(sd, spec)
    mp = om.MdxParams(dim_f, dim_t, n_fft, stem_name="Vocals", compensation=1.035)
    rng = np.random.default_rng(0)
    N = 44100 * 3 + 1234
    wave = (rng.standard_normal((2, N)) * 0.2).astype(np.float32)
    # stft / istft
    x = torch.from_numpy(wave[:, :mp.chunk_size].copy())[None]
    spec = mp.stft(x)
    assert _sha(spec) == str(pins["mdx_stft_sha"])
    assert _sha(mp.istft(spec)) == str(pins["mdx_istft_sha"])
    # full process_wave
    got = om.process_wave(wave.copy(), mp, net, 2)
    assert tuple(pins["mdx_shape"]) == got.shape == wave.shape
    assert np.abs(got.ravel()[pins["mdx_idx"]] - pins["mdx_out"]).max() < 1e-6
