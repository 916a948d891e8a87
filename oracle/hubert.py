"""TEST INFRASTRUCTURE ONLY — torch-CPU fp32 restatement of fairseq 0.12.2 `HubertModel.extract_features`
(hubert_base: conv feature extractor mode "default", post-LN transformer) as called at
vc_infer_pipeline.py:398-406.

fairseq is a third-party dependency absent from the reference repository (requirements.txt:2) -> restated from the
published architecture; cross-checked against transformers.HubertModel (tests/test_oracle_vs_reference.py);
PARITY UNPINNED against real fairseq.  State-dict names are fairseq's (SURVEY.md B9).
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]
CONV = [(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2


def pos_conv_weight(sd: SD) -> torch.Tensor:
    """weight_norm(dim=2): w = g * v / ||v||, norm over dims (0, 1) per kernel tap."""
    v, g = sd["encoder.pos_conv.0.weight_v"].float(), sd["encoder.pos_conv.0.weight_g"].float()
    return v * (g / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt())


def conv_features(sd: SD, source: torch.Tensor) -> torch.Tensor:
    """ConvFeatureExtractionModel (wav2vec2.py): [1,L] -> [1,512,T]; GroupNorm(512,512)+GELU on layer 0, GELU after."""
    x = source.unsqueeze(1)
    for i, (c, k, s) in enumerate(CONV):
        x = F.conv1d(x, sd[f"feature_extractor.conv_layers.{i}.0.weight"], stride=s)
        if i == 0:
            x = F.group_norm(x, c, sd["feature_extractor.conv_layers.0.2.weight"], sd["feature_extractor.conv_layers.0.2.bias"], 1e-5)
        x = F.gelu(x)
    return x


def extract_features(sd: SD, source: torch.Tensor, output_layer: int = 12, n_heads: int = 12) -> torch.Tensor:
    """HubertModel.extract_features(source, padding_mask=all False, mask=False, output_layer) -> [1,T,768]."""
    with torch.no_grad():
        feats = conv_features(sd, source.float()).transpose(1, 2)
        feats = F.layer_norm(feats, (feats.shape[-1],), sd["layer_norm.weight"], sd["layer_norm.bias"], 1e-5)
        x = F.linear(feats, sd["post_extract_proj.weight"], sd["post_extract_proj.bias"])
        D = x.shape[-1]
        k = sd["encoder.pos_conv.0.weight_v"].shape[-1]
        groups = D // sd["encoder.pos_conv.0.weight_v"].shape[1]
        xc = F.conv1d(x.transpose(1, 2), pos_conv_weight(sd), sd["encoder.pos_conv.0.bias"], padding=k // 2, groups=groups)
        if k % 2 == 0:
            xc = xc[:, :, :-1]                                 # SamePad
        x = x + F.gelu(xc).transpose(1, 2)
        x = F.layer_norm(x, (D,), sd["encoder.layer_norm.weight"], sd["encoder.layer_norm.bias"], 1e-5)
        dh = D // n_heads
        for i in range(output_layer):
            p = f"encoder.layers.{i}."
            q = F.linear(x, sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.q_proj.bias"]) * dh ** -0.5
            kk = F.linear(x, sd[p + "self_attn.k_proj.weight"], sd[p + "self_attn.k_proj.bias"])
            v = F.linear(x, sd[p + "self_attn.v_proj.weight"], sd[p + "self_attn.v_proj.bias"])
            B, T, _ = x.shape
            q, kk, v = (t.view(B, T, n_heads, dh).transpose(1, 2) for t in (q, kk, v))
            a = torch.softmax(q @ kk.transpose(-1, -2), dim=-1) @ v
            a = a.transpose(1, 2).reshape(B, T, D)
            a = F.linear(a, sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"])
            x = F.layer_norm(x + a, (D,), sd[p + "self_attn_layer_norm.weight"], sd[p + "self_attn_layer_norm.bias"], 1e-5)
            h = F.gelu(F.linear(x, sd[p + "fc1.weight"], sd[p + "fc1.bias"]))
            h = F.linear(h, sd[p + "fc2.weight"], sd[p + "fc2.bias"])
            x = F.layer_norm(x + h, (D,), sd[p + "final_layer_norm.weight"], sd[p + "final_layer_norm.bias"], 1e-5)
        return x


def final_proj(sd: SD, x: torch.Tensor) -> torch.Tensor:
    return F.linear(x, sd["final_proj.weight"], sd["final_proj.bias"])


def to_hf_state_dict(sd: SD) -> SD:
    """fairseq -> transformers.HubertModel key mapping (used only to cross-check this restatement)."""
    out = {}
    for i in range(len(CONV)):
        out[f"feature_extractor.conv_layers.{i}.conv.weight"] = sd[f"feature_extractor.conv_layers.{i}.0.weight"]
    out["feature_extractor.conv_layers.0.layer_norm.weight"] = sd["feature_extractor.conv_layers.0.2.weight"]
    out["feature_extractor.conv_layers.0.layer_norm.bias"] = sd["feature_extractor.conv_layers.0.2.bias"]
    out["feature_projection.layer_norm.weight"] = sd["layer_norm.weight"]
    out["feature_projection.layer_norm.bias"] = sd["layer_norm.bias"]
    out["feature_projection.projection.weight"] = sd["post_extract_proj.weight"]
    out["feature_projection.projection.bias"] = sd["post_extract_proj.bias"]
    out["encoder.pos_conv_embed.conv.bias"] = sd["encoder.pos_conv.0.bias"]
    out["encoder.pos_conv_embed.conv.parametrizations.weight.original0"] = sd["encoder.pos_conv.0.weight_g"]
    out["encoder.pos_conv_embed.conv.parametrizations.weight.original1"] = sd["encoder.pos_conv.0.weight_v"]
    out["encoder.layer_norm.weight"] = sd["encoder.layer_norm.weight"]
    out["encoder.layer_norm.bias"] = sd["encoder.layer_norm.bias"]
    n_layers = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.layers."))
    for i in range(n_layers):
        a, b = f"encoder.layers.{i}.", f"encoder.layers.{i}."
        for n in ("q", "k", "v", "out"):
            for t in ("weight", "bias"):
                out[b + f"attention.{n}_proj.{t}"] = sd[a + f"self_attn.{n}_proj.{t}"]
        for t in ("weight", "bias"):
            out[b + f"layer_norm.{t}"] = sd[a + f"self_attn_layer_norm.{t}"]
            out[b + f"feed_forward.intermediate_dense.{t}"] = sd[a + f"fc1.{t}"]
            out[b + f"feed_forward.output_dense.{t}"] = sd[a + f"fc2.{t}"]
            out[b + f"final_layer_norm.{t}"] = sd[a + f"final_layer_norm.{t}"]
    return out
