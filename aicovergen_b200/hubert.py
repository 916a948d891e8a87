"""GPU-native HuBERT-base content encoder — drop-in for the fairseq `HubertModel` object at the plug point
`model.extract_features(source=..., padding_mask=..., output_layer=...)` / `model.final_proj`
(vc_infer_pipeline.py:398-406; loaded by rvc.load_hubert, rvc.py:98-109).

7-layer strided conv front-end (tap-GEMMs over [T/s, s*C] views), GroupNorm-over-time, grouped
positional conv (16 groups x 128 taps), 12 post-LN transformer layers with materialised attention
(QK^T and PV as batched tap-GEMMs, row softmax), all through libb200vc.so on wgmma TF32.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch

from . import _ffi, ops
from . import tapgemm as tg
from .plans import ATT_SCRATCH_BYTES, PlanCache, StepGraph
from .synth import round_tf32
from .tapgemm import Epi

CONV = [(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2


class HubertB200:
    def __init__(self, state_dict: Dict[str, torch.Tensor], device: str = "cuda:0", backend: int = tg.BACKEND_TC,
                 n_heads: int = 12):
        self.device = torch.device(device)
        self.backend = backend
        self.n_heads = n_heads
        self._plans = PlanCache()
        self._load(state_dict)

    def _dev(self, t, rnd=True):
        t = t.float().contiguous()
        if rnd and self.backend == tg.BACKEND_TC:
            t = round_tf32(t)
        return t.to(self.device)

    def _load(self, sd):
        W = {}
        for i in range(len(CONV)):
            W[f"conv{i}.w"] = self._dev(tg.pack_conv1d(sd[f"feature_extractor.conv_layers.{i}.0.weight"]), i > 0)
        W["conv0.w2d"] = W["conv0.w"].permute(1, 0, 2).reshape(CONV[0][0], CONV[0][1]).contiguous()   # [512, 10] (Cin = 1)
        W["gn.g"] = self._dev(sd["feature_extractor.conv_layers.0.2.weight"], False)
        W["gn.b"] = self._dev(sd["feature_extractor.conv_layers.0.2.bias"], False)
        W["ln0.g"], W["ln0.b"] = self._dev(sd["layer_norm.weight"], False), self._dev(sd["layer_norm.bias"], False)
        W["proj.w"], W["proj.b"] = self._dev(sd["post_extract_proj.weight"]), self._dev(sd["post_extract_proj.bias"], False)
        D = sd["post_extract_proj.weight"].shape[0]
        self.dim = D
        v, g = sd["encoder.pos_conv.0.weight_v"].float(), sd["encoder.pos_conv.0.weight_g"].float()
        pw = v * (g / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt())           # [D, D/groups, k]
        self.pos_k = pw.shape[2]
        self.pos_cg = pw.shape[1]
        self.pos_groups = D // self.pos_cg
        # per group: [k, cout_g, cin_g]
        W["pos.w"] = self._dev(pw.view(self.pos_groups, self.pos_cg, self.pos_cg, self.pos_k).permute(0, 3, 1, 2))
        W["pos.b"] = self._dev(sd["encoder.pos_conv.0.bias"], False)
        W["eln.g"], W["eln.b"] = self._dev(sd["encoder.layer_norm.weight"], False), self._dev(sd["encoder.layer_norm.bias"], False)
        self.n_layers = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.layers."))
        dh = D // self.n_heads
        for i in range(self.n_layers):
            p = f"encoder.layers.{i}."
            s = dh ** -0.5   # fairseq MultiheadAttention: q = q_proj(x) * scaling
            wq, bq = sd[p + "self_attn.q_proj.weight"].float() * s, sd[p + "self_attn.q_proj.bias"].float() * s
            wk, bk = sd[p + "self_attn.k_proj.weight"].float(), sd[p + "self_attn.k_proj.bias"].float()
            W[f"l{i}.qk.w"], W[f"l{i}.qk.b"] = self._dev(torch.cat([wq, wk], 0)), self._dev(torch.cat([bq, bk], 0), False)
            W[f"l{i}.v.w"], W[f"l{i}.v.b"] = self._dev(sd[p + "self_attn.v_proj.weight"]), self._dev(sd[p + "self_attn.v_proj.bias"], False)
            W[f"l{i}.o.w"], W[f"l{i}.o.b"] = self._dev(sd[p + "self_attn.out_proj.weight"]), self._dev(sd[p + "self_attn.out_proj.bias"], False)
            W[f"l{i}.ln1.g"], W[f"l{i}.ln1.b"] = self._dev(sd[p + "self_attn_layer_norm.weight"], False), self._dev(sd[p + "self_attn_layer_norm.bias"], False)
            W[f"l{i}.fc1.w"], W[f"l{i}.fc1.b"] = self._dev(sd[p + "fc1.weight"]), self._dev(sd[p + "fc1.bias"], False)
            W[f"l{i}.fc2.w"], W[f"l{i}.fc2.b"] = self._dev(sd[p + "fc2.weight"]), self._dev(sd[p + "fc2.bias"], False)
            W[f"l{i}.ln2.g"], W[f"l{i}.ln2.b"] = self._dev(sd[p + "final_layer_norm.weight"], False), self._dev(sd[p + "final_layer_norm.bias"], False)
        if "final_proj.weight" in sd:
            W["final_proj.w"], W["final_proj.b"] = self._dev(sd["final_proj.weight"]), self._dev(sd["final_proj.bias"], False)
        self.W = W

    # ------------------------------------------------------------------ plug point
    @_ffi.on_device
    @torch.no_grad()
    def extract_features(self, source: torch.Tensor, padding_mask: Optional[torch.Tensor] = None,
                         mask: bool = False, output_layer: Optional[int] = None):
        """source [1,L] (float, on device). Returns (features [1,T,768], padding_mask) like fairseq."""
        if source.dim() != 2 or source.shape[0] != 1:
            raise ValueError("HubertB200.extract_features expects source of shape [1, L]")
        if padding_mask is not None and bool(padding_mask.any()):
            raise NotImplementedError("padded batches are not part of the RVC path (vc_infer_pipeline.py:396)")
        L = int(source.shape[1])
        nl = self.n_layers if output_layer is None else int(output_layer)
        key = (L, nl)
        plan = self._plans.get_or_build(key, lambda: _HubertPlan(self, L, nl))
        return plan.run(source), padding_mask

    @_ffi.on_device
    @torch.no_grad()
    def final_proj(self, x: torch.Tensor) -> torch.Tensor:
        """Linear 768 -> 256 used by v1 voice models (vc_infer_pipeline.py:406)."""
        W = self.W
        T = x.shape[-2]
        xin = x.reshape(T, self.dim).contiguous().float()
        out = torch.empty(T, W["final_proj.w"].shape[0], device=self.device)
        tg.linear(xin, W["final_proj.w"], out, Epi(bias=W["final_proj.b"]), self.backend, name="final_proj")()
        return out.view(*x.shape[:-1], -1)

    # fairseq modules are nn.Modules; rvc.load_hubert calls these (rvc.py:101-108)
    def to(self, *a, **k):
        return self

    def half(self):
        return self

    def float(self):
        return self

    def eval(self):
        return self


def conv_out_len(L: int) -> List[int]:
    lens = []
    for (_, k, s) in CONV:
        L = (L - k) // s + 1
        lens.append(L)
    return lens


class _HubertPlan:
    def __init__(self, m: HubertB200, L: int, n_layers: int):
        dev, W, be = m.device, m.W, m.backend
        R = be == tg.BACKEND_TC
        f32 = dict(device=dev, dtype=torch.float32)
        steps: List = []
        add = steps.append
        lens = conv_out_len(L)
        if lens[-1] < 1:
            raise ValueError(f"input of {L} samples is too short for the HuBERT front-end")
        self.wav = torch.zeros(L + 16, **f32)
        # ---- conv0 (Cin = 1, k = 10, s = 5): rows are overlapping 10-sample frames, stride 5
        T0 = lens[0]
        c0 = torch.empty(T0, 512, **f32)
        add(lambda: ops.conv1d_from1(self.wav, W["conv0.w2d"], c0, CONV[0][2], 0))
        rows_even = lambda t: t + (t % 2)
        cur = torch.zeros(rows_even(T0), 512, **f32)
        gstats = torch.zeros(2 * 512, device=dev, dtype=torch.float64)
        add(lambda cur=cur: ops.groupnorm_time(c0, W["gn.g"], W["gn.b"], cur[:T0], gstats, 1e-5, tg.ACT_GELU, R))
        # ---- conv1..6 (stride 2) through the [T/2, 2C] view
        for i in range(1, len(CONV)):
            To = lens[i]
            nxt = torch.zeros(rows_even(To), 512, **f32)
            add(tg.conv1d_strided(cur, W[f"conv{i}.w"], nxt[:To], CONV[i][2], 0,
                                  Epi(act_pre=tg.ACT_GELU, round_out=R and i < len(CONV) - 1), be, name=f"conv{i}"))
            cur = nxt
        T = lens[-1]
        self.T = T
        D, H = m.dim, m.n_heads
        dh = D // H
        feats = torch.empty(T, 512, **f32)
        add(lambda cur=cur: ops.layernorm(cur[:T], W["ln0.g"], W["ln0.b"], feats, round_out=R))
        x = torch.empty(T, D, **f32)
        add(tg.linear(feats, W["proj.w"], x, Epi(bias=W["proj.b"]), be, name="post_extract_proj"))
        # ---- grouped positional conv + GELU + residual, then LayerNorm (wav2vec2 TransformerEncoder)
        y = torch.empty(T, D, **f32)
        cg, K = m.pos_cg, m.pos_k
        for g in range(m.pos_groups):
            taps = [(g * cg, j - K // 2, 0, 0, j) for j in range(K)]
            add(tg.TapGemm(tg.view(x), tg.weights(W["pos.w"][g]), taps, (T, 1, 1), tg.out_of(y[:, g * cg:(g + 1) * cg]),
                           Epi(bias=W["pos.b"][g * cg:(g + 1) * cg], act_pre=tg.ACT_GELU, res=x[:, g * cg:(g + 1) * cg]),
                           be, name=f"pos_conv.g{g}"))
        add(lambda: ops.layernorm(y, W["eln.g"], W["eln.b"], x))
        # ---- transformer layers (post-LN)
        Tp = (T + 3) // 4 * 4
        qk = torch.empty(T, 2 * D, **f32)
        vT = torch.zeros(D, Tp, **f32)
        # Attention runs per block of QB query rows (scores [H, QB, T]); QB = T unless the scratch bound says otherwise.
        QB = min(T, max(128, (ATT_SCRATCH_BYTES // (4 * H * Tp)) // 128 * 128))
        sc = torch.zeros(H, QB, Tp, **f32)
        o = torch.empty(T, D, **f32)
        tmp = torch.empty(T, D, **f32)
        hbuf = torch.empty(T, W["l0.fc1.w"].shape[0], **f32)
        for i in range(n_layers):
            add(tg.linear(x, W[f"l{i}.qk.w"], qk, Epi(bias=W[f"l{i}.qk.b"], round_out=R), be, name=f"l{i}.qk"))
            add(tg.linear(W[f"l{i}.v.w"], x, vT[:, :T], Epi(bias=W[f"l{i}.v.b"], bias_per_row=True, round_out=R), be, name=f"l{i}.vT"))
            qh = qk[:, :D].view(T, H, dh).permute(1, 0, 2)
            kh = qk[:, D:].view(T, H, dh).permute(1, 0, 2)
            oh = o.view(T, H, dh).permute(1, 0, 2)
            for q0 in range(0, T, QB):
                nq = min(QB, T - q0)
                scb = sc[:, :nq]
                add(tg.bmm_nt(qh[:, q0:q0 + nq], kh, scb[:, :, :T], None, be, name=f"l{i}.qk^T"))
                add(lambda scb=scb: ops.softmax_rows(scb, T, round_out=R))
                add(tg.bmm_nt(scb[:, :, :T], vT.view(H, dh, Tp)[:, :, :T], oh[:, q0:q0 + nq], Epi(round_out=R), be, name=f"l{i}.pv"))
            add(tg.linear(o, W[f"l{i}.o.w"], tmp, Epi(bias=W[f"l{i}.o.b"], res=x), be, name=f"l{i}.o"))
            add(lambda i=i: ops.layernorm(tmp, W[f"l{i}.ln1.g"], W[f"l{i}.ln1.b"], x))
            add(tg.linear(x, W[f"l{i}.fc1.w"], hbuf, Epi(bias=W[f"l{i}.fc1.b"], act_pre=tg.ACT_GELU, round_out=R), be, name=f"l{i}.fc1"))
            add(tg.linear(hbuf, W[f"l{i}.fc2.w"], tmp, Epi(bias=W[f"l{i}.fc2.b"], res=x), be, name=f"l{i}.fc2"))
            add(lambda i=i: ops.layernorm(tmp, W[f"l{i}.ln2.g"], W[f"l{i}.ln2.b"], x))
        self.x = x
        self.steps = steps
        self.graph = StepGraph(steps)
        self.L = L

    def run(self, source: torch.Tensor) -> torch.Tensor:
        self.wav[:self.L].copy_(source.reshape(-1))
        self.graph()
        return self.x.view(1, self.T, -1)
