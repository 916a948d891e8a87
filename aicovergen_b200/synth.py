"""GPU-native RVC synthesizer (`net_g`): TextEncoder -> reverse flow -> NSF-HiFiGAN.

Drop-in for the reference's SynthesizerTrnMs{256,768}NSFsid at the operator plug point
`net_g.infer(feats, p_len, pitch, pitchf, sid)` (vc_infer_pipeline.py:454-465;
infer_pack/models.py:634-640, 745-751).  Everything numerical runs in libb200vc.so:
tap-GEMMs on wgmma (TF32) plus the fp32 row kernels of ops.py.  This file only
prepares weights (weight-norm folding, packing, flow Flip folding) and sequences launches.

The random draws of the reference (`randn_like` at models.py:748 and :368) are explicit
inputs (`noise_z`, `noise_src`); when omitted they are drawn on the device.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _ffi, ops
from . import tapgemm as tg
from .plans import ATT_SCRATCH_BYTES, PlanCache, StepGraph
from .tapgemm import Epi

LRELU = 0.1



def fold_weight_norm(sd: Dict[str, torch.Tensor], name: str) -> torch.Tensor:
    """w = g * v / ||v|| (norm over all dims but 0) — old-style torch weight_norm as stored in RVC checkpoints."""
    if name + ".weight" in sd:
        return sd[name + ".weight"].float()
    v, g = sd[name + ".weight_v"].float(), sd[name + ".weight_g"].float()
    return v * (g / v.flatten(1).norm(dim=1).reshape(g.shape))


def round_tf32(t: torch.Tensor) -> torch.Tensor:
    """Round-to-nearest to 10 mantissa bits so the tensor core's operand truncation is exact."""
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


# opt-in (round 2): fp16 storage of the vocoder's GEMM-only tensors (the leaky-ReLU copies and the ResBlock mid tensor) and of
# the ResBlock weights — wgmma f16, fp32 accumulate, the residual streams stay fp32.  Validated at the GEMM level only.
SYNTH_FP16 = __import__("os").environ.get("B200VC_SYNTH_FP16", "1") == "1"      # default ON from r02e (2.1e-4 abs RMS, same as TF32)


class SynthesizerB200:
    def __init__(self, cpt: dict, device="cuda:0", backend: int = tg.BACKEND_TC):
        cfg = cpt["config"]
        self.cfg = cfg
        (self.spec_channels, self.segment_size, self.inter, self.hidden, self.filter, self.n_heads,
         self.n_layers, self.ksz) = cfg[:8]
        self.rb_k, self.rb_d, self.up_r, self.up_init, self.up_k = cfg[10], cfg[11], cfg[12], cfg[13], cfg[14]
        self.gin = cfg[16]
        sr = cfg[17]
        self.sr = {"32k": 32000, "40k": 40000, "48k": 48000}.get(sr, sr)
        self.upp = int(np.prod(self.up_r))
        self.f0 = int(cpt.get("f0", 1))
        self.version = cpt.get("version", "v1")
        self.device = torch.device(device)
        self.backend = backend
        self.half_rb = bool(SYNTH_FP16 and backend == tg.BACKEND_TC)
        self.window = 10
        self._plans = PlanCache()
        self._cond_cache: Dict[int, dict] = {}
        self._load(cpt["weight"])

    # ------------------------------------------------------------------ weights
    def _dev(self, t: torch.Tensor, rnd: bool = True) -> torch.Tensor:
        t = t.float().contiguous()
        if rnd and self.backend == tg.BACKEND_TC:
            t = round_tf32(t)
        return t.to(self.device)

    def _load(self, sd: Dict[str, torch.Tensor]):
        sd = {k: v for k, v in sd.items()}
        W = {}
        H, dk = self.hidden, self.hidden // self.n_heads
        W["emb_phone.w"] = self._dev(sd["enc_p.emb_phone.weight"])
        W["emb_phone.b"] = self._dev(sd["enc_p.emb_phone.bias"], False)
        if self.f0:
            W["emb_pitch"] = self._dev(sd["enc_p.emb_pitch.weight"], False)
        for i in range(self.n_layers):
            p = f"enc_p.encoder.attn_layers.{i}."
            s = 1.0 / math.sqrt(dk)   # query scaling folded into the projection (attentions.py:233,240)
            wq, bq = sd[p + "conv_q.weight"][:, :, 0].float() * s, sd[p + "conv_q.bias"].float() * s
            wk, bk = sd[p + "conv_k.weight"][:, :, 0].float(), sd[p + "conv_k.bias"].float()
            W[f"l{i}.qk.w"] = self._dev(torch.cat([wq, wk], 0))
            W[f"l{i}.qk.b"] = self._dev(torch.cat([bq, bk], 0), False)
            W[f"l{i}.v.w"] = self._dev(sd[p + "conv_v.weight"][:, :, 0])
            W[f"l{i}.v.b"] = self._dev(sd[p + "conv_v.bias"], False)
            W[f"l{i}.o.w"] = self._dev(sd[p + "conv_o.weight"][:, :, 0])
            W[f"l{i}.o.b"] = self._dev(sd[p + "conv_o.bias"], False)
            W[f"l{i}.rel_k"] = self._dev(sd[p + "emb_rel_k"][0], False)
            W[f"l{i}.rel_v"] = self._dev(sd[p + "emb_rel_v"][0], False)
            for n in (1, 2):
                W[f"l{i}.ln{n}.g"] = self._dev(sd[f"enc_p.encoder.norm_layers_{n}.{i}.gamma"], False)
                W[f"l{i}.ln{n}.b"] = self._dev(sd[f"enc_p.encoder.norm_layers_{n}.{i}.beta"], False)
                q = f"enc_p.encoder.ffn_layers.{i}.conv_{n}."
                W[f"l{i}.ffn{n}.w"] = self._dev(tg.pack_conv1d(sd[q + "weight"]))
                W[f"l{i}.ffn{n}.b"] = self._dev(sd[q + "bias"], False)
        W["proj.w"] = self._dev(sd["enc_p.proj.weight"][:, :, 0])
        W["proj.b"] = self._dev(sd["enc_p.proj.bias"], False)
        # ---- flow: Flip() folded into the channel order of pre / post (modules.py:377-384)
        half = self.inter // 2
        for f in range(4):
            p = f"flow.flows.{2 * f}."
            pre_w, pre_b = sd[p + "pre.weight"][:, :, 0].float(), sd[p + "pre.bias"].float()
            post_w, post_b = sd[p + "post.weight"][:, :, 0].float(), sd[p + "post.bias"].float()
            W[f"f{f}.pre.w"] = self._dev(pre_w)
            W[f"f{f}.pre.w_rev"] = self._dev(pre_w.flip(1))
            W[f"f{f}.pre.b"] = self._dev(pre_b, False)
            W[f"f{f}.post.w"] = self._dev(post_w)
            W[f"f{f}.post.w_rev"] = self._dev(post_w.flip(0))
            W[f"f{f}.post.b"] = self._dev(post_b, False)
            W[f"f{f}.post.b_rev"] = self._dev(post_b.flip(0), False)
            for j in range(3):
                W[f"f{f}.in{j}.w"] = self._dev(tg.pack_conv1d(fold_weight_norm(sd, p + f"enc.in_layers.{j}")))
                W[f"f{f}.in{j}.b"] = self._dev(sd[p + f"enc.in_layers.{j}.bias"], False)
                rs_w = fold_weight_norm(sd, p + f"enc.res_skip_layers.{j}")[:, :, 0]
                rs_b = sd[p + f"enc.res_skip_layers.{j}.bias"].float()
                if j < 2:
                    W[f"f{f}.res{j}.w"], W[f"f{f}.res{j}.b"] = self._dev(rs_w[:H]), self._dev(rs_b[:H], False)
                    W[f"f{f}.skip{j}.w"], W[f"f{f}.skip{j}.b"] = self._dev(rs_w[H:]), self._dev(rs_b[H:], False)
                else:
                    W[f"f{f}.skip{j}.w"], W[f"f{f}.skip{j}.b"] = self._dev(rs_w), self._dev(rs_b, False)
            W[f"f{f}.cond.w"] = self._dev(fold_weight_norm(sd, p + "enc.cond_layer")[:, :, 0], False)
            W[f"f{f}.cond.b"] = self._dev(sd[p + "enc.cond_layer.bias"], False)
        # ---- decoder
        W["pre.w"] = self._dev(tg.pack_conv1d(sd["dec.conv_pre.weight"]))
        W["pre.b"] = self._dev(sd["dec.conv_pre.bias"], False)
        W["cond.w"] = self._dev(sd["dec.cond.weight"][:, :, 0], False)
        W["cond.b"] = self._dev(sd["dec.cond.bias"], False)
        nk = len(self.rb_k)
        for i in range(len(self.up_r)):
            W[f"up{i}.w"] = self._dev(tg.pack_convt1d(fold_weight_norm(sd, f"dec.ups.{i}")))
            W[f"up{i}.b"] = self._dev(sd[f"dec.ups.{i}.bias"], False)
            if self.f0:
                nw = sd[f"dec.noise_convs.{i}.weight"].float()          # [C, 1, k]
                W[f"nc{i}.w"] = self._dev(nw[:, 0, :].contiguous(), False)
                W[f"nc{i}.b"] = self._dev(sd[f"dec.noise_convs.{i}.bias"], False)
            for j in range(nk):
                n = i * nk + j
                for m in range(len(self.rb_d[j])):
                    for c in (1, 2):
                        q = f"dec.resblocks.{n}.convs{c}.{m}"
                        wq = tg.pack_conv1d(fold_weight_norm(sd, q))
                        W[f"rb{n}.c{c}.{m}.w"] = wq.float().contiguous().half().to(self.device) if self.half_rb else self._dev(wq)
                        W[f"rb{n}.c{c}.{m}.b"] = self._dev(sd[q + ".bias"], False)
        W["post.w"] = self._dev(sd["dec.conv_post.weight"][0].t().contiguous(), False)   # [k, C]
        W["emb_g"] = self._dev(sd["emb_g.weight"], False)
        if self.f0:
            self.lin_w = float(sd["dec.m_source.l_linear.weight"].float().reshape(-1)[0])
            self.lin_b = float(sd["dec.m_source.l_linear.bias"].float().reshape(-1)[0])
        self.W = W

    # ------------------------------------------------------------------ speaker conditioning (depends on sid only)
    def _cond(self, sid: int) -> dict:
        c = self._cond_cache.get(sid)
        if c is not None:
            return c
        W, dev = self.W, self.device
        g = W["emb_g"][sid:sid + 1].contiguous()                      # [1, gin]
        out = {}
        tmp = torch.empty(1, self.up_init, device=dev)
        tg.linear(g, W["cond.w"], tmp, Epi(bias=W["cond.b"]), backend=tg.BACKEND_SIMT)()
        out["pre.b"] = torch.empty(self.up_init, device=dev)
        ops.axpby(W["pre.b"], tmp.view(-1), out["pre.b"])
        H = self.hidden
        for f in range(4):
            cf = torch.empty(1, 2 * H * 3, device=dev)
            tg.linear(g, W[f"f{f}.cond.w"], cf, Epi(bias=W[f"f{f}.cond.b"]), backend=tg.BACKEND_SIMT)()
            for j in range(3):
                b = torch.empty(2 * H, device=dev)
                ops.axpby(W[f"f{f}.in{j}.b"], cf.view(-1)[j * 2 * H:(j + 1) * 2 * H].contiguous(), b)
                out[f"f{f}.in{j}.b"] = b
        self._cond_cache[sid] = out
        return out

    # ------------------------------------------------------------------ public plug point
    @_ffi.on_device
    @torch.no_grad()
    def infer(self, phone, phone_lengths, pitch=None, nsff0=None, sid=None, max_len=None,
              noise_z: Optional[torch.Tensor] = None, noise_src: Optional[torch.Tensor] = None):
        """Same call/return convention as the reference `infer`: returns (o [1,1,P*upp], x_mask, (z, z_p, m_p, logs_p)).
        phone [1,P,768|256] f32, pitch [1,P] i64, nsff0 [1,P] f32, sid [1] i64 (all on the CUDA device)."""
        if self.f0 and (pitch is None or nsff0 is None):
            # reference: SynthesizerTrnMs*NSFsid.infer requires pitch; the _nono variants take (phone, lengths, sid)
            raise ValueError("this checkpoint was trained with f0: pitch and nsff0 are required")
        if not self.f0 and sid is None and pitch is not None:
            sid, pitch = pitch, None   # _nono call form: infer(phone, lengths, sid)
        P = int(phone.shape[1])
        sid_i = int(sid.reshape(-1)[0].item()) if sid is not None else 0
        plan = self._plans.get_or_build(P, lambda: _Plan(self, P))
        cond = self._cond(sid_i)
        return plan.run(phone, pitch, nsff0, cond, noise_z, noise_src)


class _Plan:
    """All buffers and prepared launches for one frame count P (rebuilt only when P changes)."""

    def __init__(self, m: SynthesizerB200, P: int):
        self.m, self.P = m, P
        dev, W, be = m.device, m.W, m.backend
        H, inter, heads, dk = m.hidden, m.inter, m.n_heads, m.hidden // m.n_heads
        f32 = dict(device=dev, dtype=torch.float32)
        R = be == tg.BACKEND_TC      # round GEMM-only activations to TF32 (RN) when the tensor-core path consumes them
        steps: List = []
        add = steps.append
        in_dim = W["emb_phone.w"].shape[1]
        # ---- inputs (copied in at run time)
        self.phone = torch.empty(P, in_dim, **f32)
        self.pitch = torch.zeros(P, device=dev, dtype=torch.int64)
        self.f0 = torch.zeros(P, **f32)
        self.noise_z = torch.empty(inter, P, **f32)
        L = P * m.upp
        self.L = L
        self.noise_src = torch.empty(L, **f32)
        # per-call conditioned biases are copied into these fixed buffers so prepared launches stay valid
        self.pre_b = torch.empty(m.up_init, **f32)
        self.in_b = {(f, j): torch.empty(2 * H, **f32) for f in range(4) for j in range(3)}

        # ================= enc_p (models.py:93-108) =================
        x = torch.empty(P, H, **f32)
        if m.f0:
            emb = torch.empty(P, H, **f32)
            add(lambda: ops.gather_rows(W["emb_pitch"], self.pitch, emb))
        add(tg.linear(self.phone, W["emb_phone.w"], x,
                      Epi(bias=W["emb_phone.b"], res=emb if m.f0 else None, scale=math.sqrt(H),
                          act_post=tg.ACT_LRELU, act_post_p=LRELU), be, name="emb_phone"))
        Tp = (P + 3) // 4 * 4
        qk = torch.empty(P, 2 * H, **f32)
        vT = torch.zeros(H, Tp, **f32)
        # attention per block of QB query rows (see plans.ATT_SCRATCH_BYTES; one block by default); the relative-position band terms take
        # the block's first row as `row0`
        QB = min(P, max(128, (ATT_SCRATCH_BYTES // (4 * heads * Tp)) // 128 * 128))
        sc = torch.zeros(heads, QB, Tp, **f32)
        o = torch.empty(P, H, **f32)
        tmp = torch.empty(P, H, **f32)
        hbuf = torch.empty(P, m.filter, **f32)
        for i in range(m.n_layers):
            add(tg.linear(x, W[f"l{i}.qk.w"], qk, Epi(bias=W[f"l{i}.qk.b"], round_out=R), be, name=f"l{i}.qk"))
            # V^T = Wv X^T (+ per-row bias): operand roles swapped so the PV GEMM sees a K-major B operand
            add(tg.linear(W[f"l{i}.v.w"], x, vT[:, :P], Epi(bias=W[f"l{i}.v.b"], bias_per_row=True, round_out=R),
                          be, name=f"l{i}.vT"))
            qh = qk[:, :H].view(P, heads, dk).permute(1, 0, 2)
            kh = qk[:, H:].view(P, heads, dk).permute(1, 0, 2)
            oh = o.view(P, heads, dk).permute(1, 0, 2)
            for q0 in range(0, P, QB):
                nq = min(QB, P - q0)
                scb = sc[:, :nq]
                add(tg.bmm_nt(qh[:, q0:q0 + nq], kh, scb[:, :, :P], None, be, name=f"l{i}.qk^T"))
                add(lambda i=i, scb=scb, q0=q0: ops.softmax_rows(scb, P, q=qk, emb_rel_k=W[f"l{i}.rel_k"], window=m.window,
                                                                  round_out=R, row0=q0))
                add(tg.bmm_nt(scb[:, :, :P], vT.view(heads, dk, Tp)[:, :, :P], oh[:, q0:q0 + nq], None, be, name=f"l{i}.pv"))
                add(lambda i=i, scb=scb, q0=q0: ops.relpos_value_add(o, scb, P, W[f"l{i}.rel_v"], m.window, heads, row0=q0))
            add(tg.linear(o, W[f"l{i}.o.w"], tmp, Epi(bias=W[f"l{i}.o.b"], res=x), be, name=f"l{i}.o"))
            add(lambda i=i: ops.layernorm(tmp, W[f"l{i}.ln1.g"], W[f"l{i}.ln1.b"], x))
            add(tg.conv1d(x, W[f"l{i}.ffn1.w"], hbuf, epi=Epi(bias=W[f"l{i}.ffn1.b"], act_pre=tg.ACT_RELU, round_out=R),
                          backend=be, name=f"l{i}.ffn1"))
            add(tg.conv1d(hbuf, W[f"l{i}.ffn2.w"], tmp, epi=Epi(bias=W[f"l{i}.ffn2.b"], res=x), backend=be, name=f"l{i}.ffn2"))
            add(lambda i=i: ops.layernorm(tmp, W[f"l{i}.ln2.g"], W[f"l{i}.ln2.b"], x))
        stats = torch.empty(P, 2 * inter, **f32)
        add(tg.linear(x, W["proj.w"], stats, Epi(bias=W["proj.b"]), be, name="proj"))
        S = torch.empty(P, inter, **f32)
        self.stats, self.z_p = stats, torch.empty(P, inter, **f32)
        add(lambda: ops.zp_sample(stats, self.noise_z, self.z_p))
        add(lambda: ops.axpby(self.z_p, None, S))          # S = z_p (library op: plan steps must be recordable, see plans.StepGraph)

        # ================= reverse flow (models.py:151-152) =================
        half = inter // 2
        h = torch.empty(P, H, **f32)
        a = torch.empty(P, 2 * H, **f32)
        acts = torch.empty(P, H, **f32)
        skip = torch.empty(P, H, **f32)
        flipped = False
        for f in reversed(range(4)):
            flipped = not flipped        # Flip runs before the coupling layer in reverse order
            if flipped:                  # logical x = flip(S): x0 lives in S[:, half:] reversed
                x0, x1 = S[:, half:], S[:, :half]
                pre_w, post_w, post_b = W[f"f{f}.pre.w_rev"], W[f"f{f}.post.w_rev"], W[f"f{f}.post.b_rev"]
            else:
                x0, x1 = S[:, :half], S[:, half:]
                pre_w, post_w, post_b = W[f"f{f}.pre.w"], W[f"f{f}.post.w"], W[f"f{f}.post.b"]
            add(tg.linear(x0, pre_w, h, Epi(bias=W[f"f{f}.pre.b"]), be, name=f"f{f}.pre"))
            for j in range(3):
                add(tg.conv1d(h, W[f"f{f}.in{j}.w"], a, epi=Epi(bias=self.in_b[(f, j)]), backend=be, name=f"f{f}.in{j}"))
                add(lambda: ops.gate_tanh_sigmoid(a, acts, round_out=R))
                if j < 2:
                    add(tg.linear(acts, W[f"f{f}.res{j}.w"], h, Epi(bias=W[f"f{f}.res{j}.b"], res=h), be, name=f"f{f}.res{j}"))
                add(tg.linear(acts, W[f"f{f}.skip{j}.w"], skip,
                              Epi(bias=W[f"f{f}.skip{j}.b"], res=skip if j > 0 else None), be, name=f"f{f}.skip{j}"))
            # x1 <- x1 - post(skip)   (mean-only coupling, modules.py:457)
            add(tg.linear(skip, post_w, x1, Epi(bias=post_b, scale=-1.0, res2=x1), be, name=f"f{f}.post"))
        assert not flipped
        self.z = S

        # ================= decoder (models.py:494-516) =================
        nst = len(m.up_r)
        Ts = [P]
        for u in m.up_r:
            Ts.append(Ts[-1] * u)
        Cs = [m.up_init // (2 ** (i + 1)) for i in range(nst)]
        xl0 = torch.empty(P, m.up_init, **f32)
        add(tg.conv1d(S, W["pre.w"], xl0, epi=Epi(bias=self.pre_b, act_post=tg.ACT_LRELU, act_post_p=LRELU, round_out=R),
                      backend=be, name="conv_pre"))
        if m.f0:
            smax = max([int(np.prod(m.up_r[i + 1:])) for i in range(nst)])
            self.har_off = (smax + 3) // 4 * 4
            self.harbuf = torch.zeros(L + 2 * self.har_off + 8, **f32)
            self.cum = torch.empty(P, device=dev, dtype=torch.float64)
            har = self.harbuf[self.har_off:self.har_off + L]
            add(lambda: ops.nsf_source(self.f0, self.noise_src, har, self.cum, m.upp, m.sr, m.lin_w, m.lin_b))
        max_elems = max(Ts[i + 1] * Cs[i] for i in range(nst))
        pool = [torch.empty(max_elems, **f32) for _ in range(9)]
        hpool = {s_: torch.empty(max_elems, device=dev, dtype=torch.float16) for s_ in (1, 2, 4, 5)} if m.half_rb else {}
        prev = xl0
        nk = len(m.rb_k)
        for i in range(nst):
            T, Cc = Ts[i + 1], Cs[i]
            bufs = [(hpool[s] if s in hpool else pool[s])[:T * Cc].view(T, Cc) for s in range(9)]   # slots 1,2,4,5 = xsl, tb, xal, xbl
            sum_slot = 7 if i % 2 == 0 else 8
            xb_slot = 8 if i % 2 == 0 else 7     # the other parity slot is free inside this stage
            xs, xsl, tb, xa, xal, xbl = bufs[0], bufs[1], bufs[2], bufs[3], bufs[4], bufs[5]
            xb = bufs[6]
            Ssum = bufs[sum_slot]
            u, k = m.up_r[i], m.up_k[i]
            for op in tg.conv_transpose1d(prev, W[f"up{i}.w"], xs, u, (k - u) // 2, Epi(bias=W[f"up{i}.b"]), be, name=f"up{i}"):
                add(op)
            if m.f0:
                s = int(np.prod(m.up_r[i + 1:])) if i + 1 < nst else 1
                kk = W[f"nc{i}.w"].shape[1]
                pad = s // 2 if i + 1 < nst else 0
                # x = ups(x) + noise_conv(har) (models.py:505-507) as one write-bound row kernel; xsl = leaky_relu(x)
                add(lambda i=i, s=s, pad=pad, xs=xs, xsl=xsl: ops.conv1d_from1(
                    self.harbuf, W[f"nc{i}.w"], xs, s, self.har_off - pad, bias=W[f"nc{i}.b"], res=xs, out2=xsl,
                    act2=tg.ACT_LRELU, act2_p=LRELU, round_out2=R))
            else:
                add(lambda xs=xs, xsl=xsl: ops.act(xs, xsl, tg.ACT_LRELU, LRELU, R))
            last_stage = i == nst - 1
            for j in range(nk):
                n = i * nk + j
                cur, curl = xs, xsl
                dil = m.rb_d[j]
                outs = [(xa, xal), (xb, xbl)]
                for mm, d in enumerate(dil):
                    add(tg.conv1d(curl, W[f"rb{n}.c1.{mm}.w"], tb, dilation=d,
                                  epi=Epi(bias=W[f"rb{n}.c1.{mm}.b"], act_pre=tg.ACT_LRELU, act_pre_p=LRELU, round_out=R),
                                  backend=be, name=f"rb{n}.c1.{mm}"))
                    if mm < len(dil) - 1:
                        nxt, nxtl = outs[mm % 2]
                        add(tg.conv1d(tb, W[f"rb{n}.c2.{mm}.w"], nxt,
                                      epi=Epi(bias=W[f"rb{n}.c2.{mm}.b"], res=cur, out2=nxtl, act2=tg.ACT_LRELU,
                                              act2_p=LRELU, round_out2=R), backend=be, name=f"rb{n}.c2.{mm}"))
                        cur, curl = nxt, nxtl
                    else:
                        final = j == nk - 1
                        add(tg.conv1d(tb, W[f"rb{n}.c2.{mm}.w"], Ssum,
                                      epi=Epi(bias=W[f"rb{n}.c2.{mm}.b"], res=cur, scale=1.0 / nk,
                                              res2=Ssum if j > 0 else None,
                                              act_post=tg.ACT_LRELU if final else tg.ACT_NONE,
                                              act_post_p=(0.01 if last_stage else LRELU),
                                              round_out=R and final and not last_stage),
                                      backend=be, name=f"rb{n}.c2.{mm}"))
            prev = Ssum
        self.audio = torch.empty(L, **f32)
        add(lambda prev=prev: ops.conv1d_to1(prev, W["post.w"], self.audio, W["post.w"].shape[0] // 2, tg.ACT_TANH))
        self.steps = steps
        self.graph = StepGraph(steps)

    def run(self, phone, pitch, nsff0, cond, noise_z, noise_src):
        m, P = self.m, self.P
        self.phone.copy_(phone.reshape(P, -1))
        if m.f0:
            self.pitch.copy_(pitch.reshape(-1))
            self.f0.copy_(nsff0.reshape(-1))
        if noise_z is None:
            self.noise_z.normal_()
        else:
            self.noise_z.copy_(noise_z.reshape(m.inter, P))
        if m.f0:
            if noise_src is None:
                self.noise_src.normal_()
            else:
                self.noise_src.copy_(noise_src.reshape(-1))
        self.pre_b.copy_(cond["pre.b"])
        for (f, j), b in self.in_b.items():
            b.copy_(cond[f"f{f}.in{j}.b"])
        self.graph()
        o = self.audio.view(1, 1, -1)
        x_mask = torch.ones(1, 1, P, device=m.device)
        m_p = self.stats[:, :m.inter].t().unsqueeze(0)
        logs_p = self.stats[:, m.inter:].t().unsqueeze(0)
        return o, x_mask, (self.z.t().unsqueeze(0), self.z_p.t().unsqueeze(0), m_p, logs_p)
