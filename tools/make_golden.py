"""Generate tests/golden/*.npz by running the UNMODIFIED reference (imported with the stub recipe of
oracle/ref_import.py) on seeded synthetic checkpoints.  Needs a checkout of the reference repository:

    AICOVERGEN_REFERENCE=/path/to/AICoverGen python tools/make_golden.py [pins]
The fixtures pin (a) the oracle restatements on any machine (tests/test_golden_cpu.py) and (b) the CUDA path on
the GPU (tests/test_golden_gpu.py), and what tests/test_oracle_vs_reference.py compares with (oracle_pins.npz).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from aicovergen_b200.synthetic import (make_hubert_state_dict, make_mdx_state_dict, make_rmvpe_state_dict,  # noqa: E402
                                       make_rvc_checkpoint)
from oracle import hubert as ohub  # noqa: E402
from oracle import mdx as om  # noqa: E402
from oracle import ref_import  # noqa: E402
from refshim import HubertShim, ref_net_g, ref_rmvpe, ref_vc  # noqa: E402
from siggen import stereo_tones, vocal_like  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
os.makedirs(OUT, exist_ok=True)


def synth():
    cpt = make_rvc_checkpoint("40k", "v2", seed=1234)
    net = ref_net_g(cpt)
    P = 40
    g = torch.Generator().manual_seed(21)
    phone = torch.randn(1, P, 768, generator=g)
    pitch = torch.randint(1, 255, (1, P), generator=g)
    pitchf = (180 + 60 * torch.sin(torch.arange(P) * 0.2))[None].float()
    pitchf[:, 11:17] = 0
    torch.manual_seed(77)
    with torch.no_grad():
        o, _, (z, z_p, m_p, logs_p) = net.infer(phone, torch.tensor([P]), pitch, pitchf, torch.tensor([0]))
    np.savez_compressed(os.path.join(OUT, "synth_v2_40k.npz"), phone=phone.numpy(), pitch=pitch.numpy(), pitchf=pitchf.numpy(),
                        noise_seed=77, ckpt_seed=1234, out=o.numpy()[0, 0], m_p=m_p.numpy(), z=z.numpy())


def rmvpe():
    sd = make_rmvpe_state_dict(seed=4321)
    rm = ref_rmvpe(sd)
    x = vocal_like(1.6, seed=11)
    f0 = rm.infer_from_audio(x, 0.03)
    with torch.no_grad():
        hid = rm.mel2hidden(rm.mel_extractor(torch.from_numpy(x)[None]))[0].numpy()
    np.savez_compressed(os.path.join(OUT, "rmvpe.npz"), seconds=1.6, audio_seed=11, f0=f0, salience_argmax=hid.argmax(1), ckpt_seed=4321,
                        salience_max=hid.max(1))


def pipeline():
    hsd, rsd, cpt = make_hubert_state_dict(seed=777), make_rmvpe_state_dict(seed=4321), make_rvc_checkpoint("40k", "v2", seed=1234)
    audio = vocal_like(3.4, seed=13)
    xs = dict(x_pad=1, x_query=1, x_center=1, x_max=2)
    _, vc = ref_vc(40000, **xs)
    vc.model_rmvpe = ref_rmvpe(rsd)
    net = ref_net_g(cpt)
    torch.manual_seed(9)
    out = vc.pipeline(HubertShim(hsd), net, 0, audio.copy(), "x.wav", [0, 0, 0], 0, "rmvpe", "", 0.5, 1, 3, 40000, 0, 0.25,
                      "v2", 0.33, 128)
    np.savez_compressed(os.path.join(OUT, "vc_pipeline.npz"), seconds=3.4, audio_seed=13, out_int16=out, noise_seed=9, **{k: np.int64(v) for k, v in xs.items()})


def mdx():
    ref = ref_import.module("mdx")
    dim_f, dim_t, n_fft = 256, 16, 2048
    sd = make_mdx_state_dict(dim_f=dim_f, dim_t=dim_t, g=8, n=3, seed=2024)

    class FakeSession:
        def __init__(self, path, providers=None):
            pass

        def run(self, _, feed):
            return [om.convtdfnet(sd, torch.from_numpy(feed["input"])).numpy()]

    sys.modules["onnxruntime"].InferenceSession = FakeSession
    ref.ort.InferenceSession = FakeSession
    model = ref.MDXModel(torch.device("cpu"), dim_f=dim_f, dim_t=dim_t, n_fft=n_fft, stem_name="Vocals", compensation=1.035)
    sess = ref.MDX("fake.onnx", model, processor=-1)
    n = 44100 * 2 + 4321        # > 2 margins so both halves keep something
    wave = stereo_tones(n, seed=4)
    out = sess.process_wave(wave.copy(), 2)
    spec = model.stft(torch.from_numpy(wave[:, :model.chunk_size].copy())[None])
    np.savez_compressed(os.path.join(OUT, "mdx_small.npz"), n=n, wave_seed=4, processed=out.astype(np.float32), dim_f=dim_f, dim_t=dim_t,
                        n_fft=n_fft, ckpt_seed=2024, stft_abs_sum=float(spec.abs().sum()), spec_slice=spec[0, :, :8, :4].numpy())


def _sample_idx(n, k, seed):
    """A fixed, seeded, sorted sample of k of n positions (fixtures stay small; tests compare at these positions)."""
    return np.sort(np.random.default_rng(seed).choice(n, size=min(k, n), replace=False))


def _sha(t):
    import hashlib
    a = t.numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def pins():
    """What tests/test_oracle_vs_reference.py compares the oracle with: the reference's outputs on the same seeded inputs
    (bit-exact comparisons as SHA-256 of the reference tensor, tolerance comparisons on a seeded sample of positions)."""
    import tempfile

    from aicovergen_b200.synthetic import make_ivf_index_data
    from oracle.index import IvfFlatIndex

    z = {}
    # synth (test_synth_oracle_matches_reference)
    cpt = make_rvc_checkpoint("40k", "v2")
    net = ref_net_g(cpt)
    P = 48
    g = torch.Generator().manual_seed(1)
    phone = torch.randn(1, P, 768, generator=g)
    pitch = torch.randint(1, 255, (1, P), generator=g)
    pitchf = torch.rand(1, P, generator=g) * 300 + 80
    pitchf[:, 7:15] = 0
    torch.manual_seed(11)
    with torch.no_grad():
        o_ref = net.infer(phone, torch.tensor([P]), pitch, pitchf, torch.tensor([0]))[0].numpy().ravel()
    z["synth_idx"] = _sample_idx(o_ref.size, 6000, 1)
    z["synth_out"] = o_ref[z["synth_idx"]]
    z["synth_n"] = o_ref.size
    # parameter names / shapes the reference modules expect (test_synthetic_checkpoints_load_strictly_in_reference)
    m = ref_import.module("infer_pack.models")
    for key in ("40k", "48k_v2", "32k"):
        c = make_rvc_checkpoint(key, "v2")
        n_ = m.SynthesizerTrnMs768NSFsid(*c["config"], is_half=False)
        del n_.enc_q
        sd = n_.state_dict()
        z[f"params_{key}"] = np.array([f"{k}:{tuple(v.shape)}" for k, v in sorted(sd.items())])
    r = ref_import.module("rmvpe")
    z["params_rmvpe"] = np.array([f"{k}:{tuple(v.shape)}" for k, v in sorted(r.E2E(4, 1, (2, 2)).state_dict().items())])
    # rmvpe (test_rmvpe_oracle_matches_reference)
    from oracle import rmvpe as orm
    rsd = make_rmvpe_state_dict()
    rm = ref_rmvpe(rsd)
    x = vocal_like(2.5)
    z["rmvpe_f0"] = rm.infer_from_audio(x, 0.03)
    with torch.no_grad():
        mel = rm.mel_extractor(torch.from_numpy(x)[None])
        h = rm.mel2hidden(mel)[0].numpy()
    z["rmvpe_mel_sha"] = _sha(mel)
    hs = h[::6].copy()                    # decode is exact given the same salience: every 6th frame is enough to pin it
    z["rmvpe_salience"] = hs
    z["rmvpe_decode"] = rm.decode(hs.copy(), 0.03)
    # pipeline (test_pipeline_oracle_matches_reference), without and with an index
    hsd = make_hubert_state_dict(layers=2)
    audio = vocal_like(5.3)
    xs = dict(x_pad=1, x_query=1, x_center=2, x_max=3)
    for with_index in (False, True):
        file_index = ""
        vmod, vc = ref_vc(40000, **xs)
        if with_index:
            base = ohub.extract_features(hsd, torch.from_numpy(vocal_like(3.0, seed=3))[None], 2)[0]
            cent, vecs = make_ivf_index_data(base, n_total=2000, nlist=40)
            index = IvfFlatIndex(cent, vecs)
            tmp = tempfile.NamedTemporaryFile(suffix=".index", delete=False)
            tmp.close()
            file_index = tmp.name
            sys.modules["faiss"].read_index = lambda p_: index
        vc.model_rmvpe = ref_rmvpe(rsd)

        class Shim(HubertShim):
            def extract_features(self, source, padding_mask, output_layer):
                return (ohub.extract_features(self.sd, source.float(), 2), padding_mask)
        net_g = ref_net_g(cpt)
        torch.manual_seed(5)
        out = vc.pipeline(Shim(hsd), net_g, 0, audio.copy(), "x.wav", [0, 0, 0], 0, "rmvpe", file_index,
                          0.5, 1, 3, 40000, 0, 0.25, "v2", 0.33, 128)
        if with_index:
            os.unlink(file_index)
        k = f"pipeline_{int(with_index)}"
        z[k + "_n"] = out.size
        z[k + "_idx"] = _sample_idx(out.size, 12000, 2)
        z[k + "_out"] = out[z[k + "_idx"]]
    # mdx (test_mdx_oracle_matches_reference)
    ref = ref_import.module("mdx")
    dim_f, dim_t, n_fft = 256, 16, 2048
    sd = make_mdx_state_dict(dim_f=dim_f, dim_t=dim_t, g=8, n=3)

    class FakeSession:
        def __init__(self, path, providers=None):
            pass

        def run(self, _, feed):
            return [om.convtdfnet(sd, torch.from_numpy(feed["input"])).numpy()]

    sys.modules["onnxruntime"].InferenceSession = FakeSession
    ref.ort.InferenceSession = FakeSession
    model = ref.MDXModel(torch.device("cpu"), dim_f=dim_f, dim_t=dim_t, n_fft=n_fft, stem_name="Vocals", compensation=1.035)
    sess = ref.MDX("fake.onnx", model, processor=-1)
    rng = np.random.default_rng(0)
    N = 44100 * 3 + 1234
    wave = (rng.standard_normal((2, N)) * 0.2).astype(np.float32)
    xc = torch.from_numpy(wave[:, :model.chunk_size].copy())[None]
    spec = model.stft(xc)
    z["mdx_stft_sha"] = _sha(spec)
    z["mdx_istft_sha"] = _sha(model.istft(spec))
    out = sess.process_wave(wave.copy(), 2)
    z["mdx_shape"] = np.array(out.shape)
    z["mdx_idx"] = _sample_idx(out.size, 12000, 3)
    z["mdx_out"] = out.ravel()[z["mdx_idx"]]
    np.savez_compressed(os.path.join(OUT, "oracle_pins.npz"), **z)


if __name__ == "__main__":
    if sys.argv[1:] == ["pins"]:
        pins()
    else:
        synth()
        rmvpe()
        pipeline()
        mdx()
        pins()
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))
