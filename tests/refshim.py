"""Helpers to run the UNMODIFIED reference (oracle/ref_import.py) with duck-typed operators, for tools/make_golden.py.
Only usable where a reference checkout is available. TEST INFRASTRUCTURE ONLY."""
import types

import numpy as np
import torch

from oracle import hubert as ohub
from oracle import ref_import


class HubertShim:
    """Duck-typed fairseq HubertModel backed by the oracle restatement (fairseq itself is not installable)."""

    def __init__(self, sd):
        self.sd = sd

    def extract_features(self, source, padding_mask, output_layer):
        return (ohub.extract_features(self.sd, source.float(), output_layer), padding_mask)

    def final_proj(self, x):
        return ohub.final_proj(self.sd, x)


def ref_net_g(cpt):
    m = ref_import.module("infer_pack.models")
    cls = m.SynthesizerTrnMs768NSFsid if cpt.get("version", "v1") == "v2" else m.SynthesizerTrnMs256NSFsid
    net = cls(*cpt["config"], is_half=False)
    del net.enc_q
    net.load_state_dict(cpt["weight"], strict=False)
    return net.eval().float()


def ref_rmvpe(sd):
    r = ref_import.module("rmvpe")
    model = r.E2E(4, 1, (2, 2))
    model.load_state_dict(sd)
    model.eval()
    rm = r.RMVPE.__new__(r.RMVPE)
    rm.model, rm.is_half, rm.device, rm.resample_kernel = model, False, "cpu", {}
    rm.mel_extractor = r.MelSpectrogram(False, 128, 16000, 1024, 160, None, 30, 8000)
    rm.cents_mapping = np.pad(20 * np.arange(360) + 1997.3794084376191, (4, 4))
    return rm


def ref_vc(tgt_sr, x_pad=3, x_query=10, x_center=60, x_max=65):
    v = ref_import.module("vc_infer_pipeline")
    cfg = types.SimpleNamespace(device="cpu", is_half=False, x_pad=x_pad, x_query=x_query, x_center=x_center, x_max=x_max)
    return v, v.VC(tgt_sr, cfg)


from siggen import vocal_like  # noqa: E402,F401
