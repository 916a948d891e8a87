"""The reference's own file-level call surface, executed end to end on the GPU with synthetic model FILES in the formats
the reference loads (closes SURVEY.md §8 rows a1-a4, a17, a21, a22):

    rvc.Config -> rvc.load_hubert(path) -> rvc.get_vc(path) -> rvc.rvc_infer(16 positional args)      rvc.py:20-151
    mdx.run_mdx(model_params, out_dir, model.onnx, wav, ...) incl. MDX.get_hash -> model_data lookup  mdx.py:238-287, 81-90
    main.song_cover_pipeline(song, voice_model, pitch_change, keep_files, ...)                        main.py:236-316

Each file-level result is compared with the array-level path on the same inputs."""
import json
import os
import sys

import numpy as np
import pytest
import torch
from scipy.io import wavfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from siggen import song_44k, vocal_like  # noqa: E402

from aicovergen_b200.synthetic import (make_hubert_state_dict, make_ivf_index_data, make_mdx_trained_like,  # noqa: E402
                                       make_rmvpe_trained_like, make_rvc_checkpoint)

pytestmark = pytest.mark.gpu

# small-geometry stand-ins for the three separation models (same code path as the 3072-bin ones; full-size geometry is
# covered by tests/test_baseline_configs_gpu.py): name -> (dim_f, log2 dim_t, n_fft, stem, compensate)
SMALL_MDX = {
    "UVR-MDX-NET-Voc_FT": (256, 5, 2048, "Vocals", 1.021),
    "UVR_MDXNET_KARA_2": (128, 5, 2048, "Instrumental", 1.035),
    "Reverb_HQ_By_FoxJoy": (256, 6, 2048, "Other", 1.035),
}


def _write_models(root):
    """mdxnet_models/*.onnx + model_data.json (shipped entries + the synthetic files' md5 tails), rvc_models/hubert_base.pt,
    rmvpe.pt, <voice>/<voice>.pth + added_IVF*.index — exactly the layout main.py:19-21, 150-163 expects."""
    from aicovergen_b200 import onnx_io
    from aicovergen_b200.faiss_io import write_ivfflat
    from aicovergen_b200.mdx import MDX
    from oracle import hubert as ohub
    from oracle.index import IvfFlatIndex

    mdx_dir, rvc_dir = os.path.join(root, "mdxnet_models"), os.path.join(root, "rvc_models")
    os.makedirs(mdx_dir), os.makedirs(os.path.join(rvc_dir, "Synth"))
    repo_json = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mdxnet_models", "model_data.json")
    with open(repo_json) as f:
        params = json.load(f)
    assert len(params) >= 50 and params["2cdd429caac38f0194b133884160f2c6"]["mdx_dim_f_set"] == 3072     # shipped config data
    sds = {}
    for i, (name, (dim_f, lt, n_fft, stem, comp)) in enumerate(SMALL_MDX.items()):
        sd = make_mdx_trained_like(dim_f, 2 ** lt, n_fft, seed=31 + i, g=8, n=3)
        path = os.path.join(mdx_dir, name + ".onnx")
        onnx_io.write_convtdfnet_onnx(path, sd, fold_bn=True)
        h = MDX.get_hash(path)
        assert h not in params
        params[h] = {"compensate": comp, "mdx_dim_f_set": dim_f, "mdx_dim_t_set": lt, "mdx_n_fft_scale_set": n_fft,
                     "primary_stem": stem}
        sds[name] = sd
    with open(os.path.join(mdx_dir, "model_data.json"), "w") as f:
        json.dump(params, f)
    hsd, rsd, cpt = make_hubert_state_dict(), make_rmvpe_trained_like(), make_rvc_checkpoint("40k", "v2")
    torch.save({"model": hsd, "cfg": None, "args": None}, os.path.join(rvc_dir, "hubert_base.pt"))      # fairseq checkpoint layout
    torch.save(rsd, os.path.join(rvc_dir, "rmvpe.pt"))
    half_cpt = dict(cpt, weight={k: (v.half() if v.is_floating_point() else v) for k, v in cpt["weight"].items()})
    torch.save(half_cpt, os.path.join(rvc_dir, "Synth", "Synth.pth"))                                 # RVC ships fp16 weights
    base = ohub.extract_features(hsd, torch.from_numpy(vocal_like(4.0, seed=3))[None], 12)[0]
    cent, vecs = make_ivf_index_data(base, n_total=4000, nlist=64, lloyd=False)
    idx = IvfFlatIndex(cent, vecs)
    write_ivfflat(os.path.join(rvc_dir, "Synth", "added_IVF64_Flat_nprobe_1_Synth_v2.index"), cent, vecs, idx.assign)
    return mdx_dir, rvc_dir, params, sds, (hsd, rsd, half_cpt)


def _read(path):
    sr, d = wavfile.read(path)
    return sr, d


def test_file_level_call_surface(tmp_path, monkeypatch):
    from oracle import dsp as odsp
    from aicovergen_b200 import main as bmain
    from aicovergen_b200 import mdx as bmdx
    from aicovergen_b200 import rvc as brvc

    root = str(tmp_path)
    mdx_dir, rvc_dir, params, sds, (hsd, rsd, cpt) = _write_models(root)
    song = song_44k(7.0, seed=3)
    song_path = os.path.join(root, "My Song.wav")
    wavfile.write(song_path, 44100, np.rint(song.T * 32767).astype(np.int16))

    # ---------------- mdx.run_mdx: 11-argument signature, hash lookup, two wav paths --------------------------------
    out_dir = os.path.join(root, "stems")
    os.makedirs(out_dir)
    name = "UVR-MDX-NET-Voc_FT"
    voc_path, inst_path = bmdx.run_mdx(params, out_dir, os.path.join(mdx_dir, name + ".onnx"), song_path, denoise=True, keep_orig=True)
    assert os.path.basename(voc_path) == "My Song_Vocals.wav" and os.path.basename(inst_path) == "My Song_Instrumental.wav"
    dim_f, lt, n_fft, stem, comp = SMALL_MDX[name]
    wave, sr = bmdx._read_wav_44k(song_path)
    weights = bmdx.load_mdx_weights(os.path.join(mdx_dir, name + ".onnx"), 2 ** lt)          # same file -> bit-identical network
    assert [int(v) for v in weights["_meta"]] == [int(v) for v in sds[name]["_meta"]]
    sess = bmdx.MDX(weights, bmdx.MDXModel("cuda:0", dim_f, 2 ** lt, n_fft, stem_name=stem, compensation=comp), 0)
    main_a, inv_a = bmdx.run_mdx_arrays(sess, wave, denoise=True, m_threads=2)
    assert np.isfinite(main_a).all() and np.isfinite(inv_a).all() and np.abs(main_a).max() > 1e-3
    for path, arr in ((voc_path, main_a), (inst_path, inv_a)):
        sr_f, d = _read(path)
        want = odsp.pcm16_soundfile(arr.T)
        assert sr_f == 44100 and d.shape == want.shape
        assert np.array_equal(d, want), path
    with pytest.raises(KeyError):                                    # unknown hash: the reference dies on model_params.get -> None
        bmdx.run_mdx({}, out_dir, os.path.join(mdx_dir, name + ".onnx"), song_path)

    # ---------------- rvc.Config / load_hubert / get_vc / rvc_infer --------------------------------------------------
    config = brvc.Config("cuda:0", True)
    assert (config.x_pad, config.x_query, config.x_center, config.x_max) == (3, 10, 60, 65)
    # rvc.py:53-60, 89: whole GiB of the device, rounded as the reference rounds; > 4 GiB selects the (3, 10, 60, 65) segmentation
    gib = int(torch.cuda.get_device_properties(0).total_memory / 1024 / 1024 / 1024 + 0.4)
    assert config.n_cpu > 0 and config.gpu_mem == gib and config.gpu_mem > 4 and config.device == "cuda:0"
    hubert = brvc.load_hubert("cuda:0", config.is_half, os.path.join(rvc_dir, "hubert_base.pt"))
    cpt_l, version, net_g, tgt_sr, vc = brvc.get_vc("cuda:0", config.is_half, config, os.path.join(rvc_dir, "Synth", "Synth.pth"))
    assert (version, tgt_sr, cpt_l["config"][-3]) == ("v2", 40000, 109) and isinstance(vc, brvc.VC)
    with pytest.raises(ValueError):
        brvc.get_vc("cuda:0", True, config, {"weights": {}})
    index_path = os.path.join(rvc_dir, "Synth", "added_IVF64_Flat_nprobe_1_Synth_v2.index")
    monkeypatch.setattr(brvc, "BASE_DIR", root)                      # VC.get_f0 loads rvc_models/rmvpe.pt from BASE_DIR (:323-328)
    vc.set_noise_seed(5)
    out_wav = os.path.join(root, "converted.wav")
    brvc.rvc_infer(index_path, 0.5, voc_path, out_wav, 0, "rmvpe", cpt_l, version, net_g, 3, tgt_sr, 0.25, 0.33, 128, vc, hubert)
    assert hasattr(vc, "model_rmvpe"), "rmvpe.pt must have been loaded lazily from rvc_models/"
    sr_o, conv = _read(out_wav)
    audio = brvc.load_audio(voc_path, 16000)
    vc.set_noise_seed(5)
    direct = vc.pipeline(hubert, net_g, 0, audio, voc_path, [0, 0, 0], 0, "rmvpe", index_path, 0.5, 1, 3, tgt_sr, 0, 0.25, version, 0.33, 128)
    assert sr_o == 40000 and conv.dtype == np.int16 and np.array_equal(conv, direct)
    assert abs(conv.shape[0] - len(audio) * 2.5) < 1000
    assert np.abs(conv).max() > 100, "silent conversion"

    # ---------------- main.song_cover_pipeline (21-argument signature; positional like webui.py:234-239) ------------
    monkeypatch.setattr(bmain, "mdxnet_models_dir", mdx_dir)
    monkeypatch.setattr(bmain, "rvc_models_dir", rvc_dir)
    monkeypatch.setattr(bmain, "output_dir", os.path.join(root, "song_output"))
    cover_path = bmain.song_cover_pipeline(song_path, "Synth", 0, True, 0, 0, 0, 0, 0.5, 3, 0.25, "rmvpe", 128, 0.33, 0, 0.15, 0.2,
                                           0.8, 0.7, "wav")
    assert os.path.exists(cover_path) and cover_path.endswith("My Song (Synth Ver).wav")
    song_dir = os.path.dirname(cover_path)
    files = sorted(os.listdir(song_dir))
    for suffix in ("_Vocals.wav", "_Instrumental.wav", "_Vocals_Main.wav", "_Vocals_Backup.wav", "_Vocals_Main_DeReverb.wav"):
        assert any(f.endswith(suffix) for f in files), (suffix, files)             # main.py:166-190 naming
    sr_c, cover = _read(cover_path)
    assert sr_c == 44100 and cover.ndim == 2 and cover.shape[1] == 2 and abs(cover.shape[0] - song.shape[1]) <= 4410
    assert np.abs(cover.astype(np.int32)).max() > 500
    # effects (main.py:206-226): the kept `_mixed.wav` is the converted vocal through high-pass, compressor and reverb
    mixed = [f for f in files if "_Synth_p0_i0.5_fr3_rms0.25_pro0.33_rmvpe" in f and f.endswith("_mixed.wav")]
    assert len(mixed) == 1, files
    from oracle import effects as oeff
    from oracle import mixdown as omix
    sr_raw, raw = _read(os.path.join(song_dir, mixed[0].replace("_mixed.wav", ".wav")))
    sr_a, a = _read(os.path.join(song_dir, mixed[0]))
    want_fx, _ = oeff.add_audio_effects(raw, sr_raw, 0.15, 0.2, 0.8, 0.7)
    assert sr_a == sr_raw == 40000 and a.shape == raw.shape
    d = np.abs(a.astype(np.int32) - want_fx.astype(np.int32))
    assert d.max() <= 1 and (d > 0).mean() < 0.02 and not np.array_equal(a, raw)
    # mix (main.py:229-233): the cover is pydub's gain / overlay of the three kept files, bit for bit
    b = _read([os.path.join(song_dir, f) for f in files if f.endswith("_Vocals_Backup.wav")][0])[1]
    c = _read([os.path.join(song_dir, f) for f in files if f.endswith("_Instrumental.wav")][0])[1]
    want, rate = omix.combine_audio(a, sr_a, b, 44100, c, 44100)
    assert rate == 44100 and np.array_equal(cover, want)
    # second call reuses the cached stems and the cached conversion (main.py:271-296) and returns the same path
    assert bmain.song_cover_pipeline(song_path, "Synth", 0, False, 0, 0, 0, 0, 0.5, 3, 0.25, "rmvpe", 128, 0.33, 0, 0.15, 0.2,
                                     0.8, 0.7, "wav") == cover_path
    # unsupported options are refused BEFORE any work (no new song directory appears)
    other = os.path.join(root, "Other.wav")
    wavfile.write(other, 44100, np.rint(song.T[:44100] * 32767).astype(np.int16))
    before = set(os.listdir(bmain.output_dir))
    with pytest.raises(Exception, match="pitch_change_all"):
        bmain.song_cover_pipeline(other, "Synth", 0, True, 0, 0, 0, 0, 0.5, 3, 0.25, "rmvpe", 128, 0.33, 2)
    with pytest.raises(Exception, match="f0_method"):
        bmain.song_cover_pipeline(other, "Synth", 0, True, f0_method="harvest")
    assert set(os.listdir(bmain.output_dir)) == before
