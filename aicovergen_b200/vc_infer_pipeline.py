"""Host mirror of the reference's RVC inference driver (src/vc_infer_pipeline.py) over the GPU operators.

Same class, method names, argument order and return types as the reference (`VC(tgt_sr, config)`,
`VC.pipeline(model, net_g, sid, audio, input_audio_path, times, f0_up_key, f0_method, file_index,
index_rate, if_f0, filter_radius, tgt_sr, resample_sr, rms_mix_rate, version, protect,
crepe_hop_length, f0_file=None) -> np.int16[...]`, vc_infer_pipeline.py:474-653), so `rvc.rvc_infer`
and `main.song_cover_pipeline` keep working unchanged.  What differs is where the arithmetic runs:
HuBERT / index lookup / synthesizer / rmvpe are the libb200vc.so operators and segment audio stays in
HBM between them (the reference hops D2H/H2D around faiss and after every segment).

Extension (not in the reference): `vc.set_noise_seed(seed)` makes the synthesizer's random draws replay
the CPU stream `torch.manual_seed(seed)` would give the reference, for parity tests.
"""
from __future__ import annotations

import os
import traceback
from time import time as ttime
from typing import Optional

import numpy as np
import torch
from scipy import signal

from . import _ffi, ops
from .index import IvfIndexB200, read_index

# rmvpe F0 of the whole utterance on a side stream, overlapped with the HuBERT / index half of the segments (the synthesizer
# half needs the F0).  B200VC_F0_OVERLAP=0: the reference's order (F0 first, then the segments one after the other).
F0_OVERLAP = os.environ.get("B200VC_F0_OVERLAP", "1") == "1"

# 5th-order Butterworth high-pass at 48 Hz for 16 kHz input (vc_infer_pipeline.py:22)
bh, ah = signal.butter(N=5, Wn=48, btype="high", fs=16000)


class VC(object):
    def __init__(self, tgt_sr, config):
        self.x_pad, self.x_query, self.x_center, self.x_max, self.is_half = (
            config.x_pad, config.x_query, config.x_center, config.x_max, config.is_half)
        self.sr = 16000                              # HuBERT input rate
        self.window = 160                            # samples per F0 frame
        self.t_pad = self.sr * self.x_pad            # reflect context each side of a segment
        self.t_pad_tgt = tgt_sr * self.x_pad
        self.t_pad2 = self.t_pad * 2
        self.t_query = self.sr * self.x_query        # +- search range around each nominal cut
        self.t_center = self.sr * self.x_center      # nominal cut spacing
        self.t_max = self.sr * self.x_max            # below this no cutting
        self.device = config.device
        self._noise_gen: Optional[torch.Generator] = None
        self.keep_float = False      # tests: keep the float waveform before/after the RMS mix
        self.exact_hpf = False       # True: scipy.signal.filtfilt on the host (the reference's exact ba-form numerics)
        self.return_device = False   # extension: pipeline() returns the int16 utterance as a device tensor (no D2H)
        self.group = None            # extension: torch.distributed group -> one utterance's segments are shared by its ranks

    # ------------------------------------------------------------------ extension for parity tests
    def set_noise_seed(self, seed: Optional[int]):
        self._noise_gen = None if seed is None else torch.Generator().manual_seed(int(seed))

    def _draw_noise(self, net_g, P, upload=True):
        """Replays the reference's draw order inside net_g.infer (models.py:748, :337, :368).  upload=False only advances
        the stream (segments another rank converts)."""
        if self._noise_gen is None:
            return None, None
        g = self._noise_gen
        nz = torch.randn(1, net_g.inter, P, generator=g)
        ns = None
        if net_g.f0:                     # the *_nono models draw randn_like(m_p) only (models.py:847-853)
            _ = torch.rand(1, 1, generator=g)
            ns = torch.randn(1, P * net_g.upp, 1, generator=g)
        if not upload:
            return None, None
        dev = self.device
        return nz.to(dev), (None if ns is None else ns.to(dev))

    # ------------------------------------------------------------------ F0
    def get_f0_crepe_computation(self, x, f0_min, f0_max, p_len, hop_length=160, model="full"):
        """vc_infer_pipeline.py:96-137 with `torchcrepe.predict` replaced by CrepeB200.predict (same arguments: 16 kHz,
        `hop_length`, fmin/fmax, model 'full', viterbi decoder, pad=True; the reference's batch_size only bounds memory)."""
        if model != "full":
            raise NotImplementedError("only torchcrepe's 'full' model is built")
        if not hasattr(self, "model_crepe"):
            from .crepe import CrepeB200
            from .rvc import BASE_DIR
            sd = torch.load(os.path.join(BASE_DIR, "rvc_models", "crepe_full.pth"), map_location="cpu")   # torchcrepe/assets/full.pth
            self.model_crepe = CrepeB200(sd, device=self.device)
        x = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
        x = x.astype(np.float32)
        x /= np.quantile(np.abs(x), 0.999)
        pitch = self.model_crepe.predict(x, self.sr, hop_length, f0_min, f0_max, dither_seed=getattr(self, "crepe_dither_seed", None),
                                         dither=getattr(self, "crepe_dither", True))
        p_len = p_len or x.shape[0] // hop_length
        source = np.array(pitch, dtype=np.float32)
        source[source < 0.001] = np.nan
        target = np.interp(np.arange(0, len(source) * p_len, len(source)) / p_len, np.arange(0, len(source)), source)
        return np.nan_to_num(target)

    def get_f0(self, input_audio_path, x, p_len, f0_up_key, f0_method, filter_radius, crepe_hop_length, inp_f0=None):
        """rmvpe branch of the reference (vc_infer_pipeline.py:262-278, 322-329, 346-370)."""
        f0_min, f0_max = 50, 1100
        f0_mel_min = 1127 * np.log(1 + f0_min / 700)
        f0_mel_max = 1127 * np.log(1 + f0_max / 700)
        if f0_method == "rmvpe":
            if not hasattr(self, "model_rmvpe"):
                from .rmvpe import RMVPEB200
                from .rvc import BASE_DIR
                self.model_rmvpe = RMVPEB200(os.path.join(BASE_DIR, "rvc_models", "rmvpe.pt"), is_half=self.is_half,
                                             device=self.device)
            if isinstance(x, torch.Tensor) and not hasattr(self.model_rmvpe, "infer_from_audio_device"):
                x = x.cpu().numpy()          # a reference-style RMVPE object was injected: it takes numpy
            f0 = self.model_rmvpe.infer_from_audio(x, thred=0.03)
        elif f0_method == "mangio-crepe":
            f0 = self.get_f0_crepe_computation(x, f0_min, f0_max, p_len, crepe_hop_length)
        else:
            raise NotImplementedError(
                f"f0_method={f0_method!r}: 'rmvpe' and 'mangio-crepe' run on the GPU path (pm / harvest / dio / pyin are CPU "
                "libraries outside the hot path; crepe-tiny and the hybrid methods are not built)")
        return self._coarse_from_f0(f0, f0_up_key, inp_f0)

    def _coarse_from_f0(self, f0, f0_up_key, inp_f0=None):
        """Transposition, optional f0-file override and the mel quantisation to 1..255 (vc_infer_pipeline.py:322-370), host numpy."""
        f0_min, f0_max = 50, 1100
        f0_mel_min = 1127 * np.log(1 + f0_min / 700)
        f0_mel_max = 1127 * np.log(1 + f0_max / 700)
        f0 *= pow(2, f0_up_key / 12)
        tf0 = self.sr // self.window
        if inp_f0 is not None:
            delta_t = np.round((inp_f0[:, 0].max() - inp_f0[:, 0].min()) * tf0 + 1).astype("int16")
            replace_f0 = np.interp(list(range(delta_t)), inp_f0[:, 0] * 100, inp_f0[:, 1])
            shape = f0[self.x_pad * tf0: self.x_pad * tf0 + len(replace_f0)].shape[0]
            f0[self.x_pad * tf0: self.x_pad * tf0 + len(replace_f0)] = replace_f0[:shape]
        f0bak = f0.copy()
        f0_mel = 1127 * np.log(1 + f0 / 700)
        f0_mel[f0_mel > 0] = (f0_mel[f0_mel > 0] - f0_mel_min) * 254 / (f0_mel_max - f0_mel_min) + 1
        f0_mel[f0_mel <= 1] = 1
        f0_mel[f0_mel > 255] = 255
        f0_coarse = np.rint(f0_mel).astype(int)
        return f0_coarse, f0bak

    # ------------------------------------------------------------------ one segment
    def vc(self, model, net_g, sid, audio0, pitch, pitchf, times, index, big_npy, index_rate, version, protect):
        """Returns the converted segment as a float32 DEVICE tensor (the reference returns numpy; pipeline()
        keeps segments in HBM until the final concat)."""
        has_f0 = pitch is not None and pitchf is not None
        half = self._vc_features(model, audio0, times, index, big_npy, index_rate, version, protect < 0.5 and has_f0)
        return self._vc_synth(net_g, sid, half, pitch, pitchf, times, protect)

    def _vc_features(self, model, audio0, times, index, big_npy, index_rate, version, keep_raw, own=False):
        """First half of VC.vc (vc_infer_pipeline.py:385-431): HuBERT features (+ final_proj for v1) and the index blend;
        nothing here needs the F0.  own=True: the returned tensors do not alias per-shape plan buffers (the caller keeps the
        halves of several segments alive at once)."""
        dev = self.device
        feats = torch.from_numpy(np.ascontiguousarray(audio0)).float() if isinstance(audio0, np.ndarray) else audio0.float()
        if feats.dim() == 2:
            feats = feats.mean(-1)
        assert feats.dim() == 1, feats.dim()
        n_in = feats.shape[0]
        feats = feats.view(1, -1).to(dev)
        padding_mask = torch.zeros(feats.shape, dtype=torch.bool)          # host-side: checking it must not sync the stream
        t0 = ttime()
        logits = model.extract_features(source=feats, padding_mask=padding_mask, output_layer=9 if version == "v1" else 12)
        feats = model.final_proj(logits[0]) if version == "v1" else logits[0]
        f2d = feats[0]                                             # [T, C]
        feats0 = f2d.clone() if keep_raw else None
        if index is not None and big_npy is not None and index_rate != 0:
            f2d = index.search_blend(f2d, index_rate)
        if own:
            f2d = f2d.clone()
        times[0] += ttime() - t0
        return f2d, feats0, n_in

    def _vc_synth(self, net_g, sid, half, pitch, pitchf, times, protect):
        """Second half of VC.vc (vc_infer_pipeline.py:432-470): 2x feature upsampling with the protect blend, synthesizer."""
        dev = self.device
        f2d, feats0, n_in = half
        has_f0 = pitch is not None and pitchf is not None
        do_protect = protect < 0.5 and has_f0
        t1 = ttime()
        p_len = n_in // self.window
        if 2 * f2d.shape[0] < p_len:
            p_len = 2 * f2d.shape[0]
        if has_f0:
            pitch = pitch[:, :p_len]
            pitchf = pitchf[:, :p_len]
        up = torch.empty(p_len, f2d.shape[1], device=dev)
        ops.upsample2_protect(f2d.contiguous(), feats0, pitchf.reshape(-1).contiguous() if has_f0 else None, up,
                              protect, do_protect)
        p_len_t = torch.tensor([p_len], device=dev).long()
        nz, ns = self._draw_noise(net_g, p_len)
        if has_f0:
            audio1 = net_g.infer(up.unsqueeze(0), p_len_t, pitch, pitchf, sid, noise_z=nz, noise_src=ns)[0][0, 0]
        else:
            audio1 = net_g.infer(up.unsqueeze(0), p_len_t, sid, noise_z=nz)[0][0, 0]
        times[2] += ttime() - t1
        return audio1

    # ------------------------------------------------------------------ segment sharding (extension)
    def _segment_frames(self, n_in: int) -> int:
        """p_len of a segment of n_in samples: min(n_in // window, 2 * HuBERT frames) (vc_infer_pipeline.py:433-441)."""
        from .hubert import conv_out_len
        return min(n_in // self.window, 2 * conv_out_len(n_in)[-1])

    def _gather_segments(self, outs, seg_samples, net_g, world, rank):
        """All-gather of the converted segments (<= 38 MB for a 4-min song): round k exchanges segments k*world .. k*world +
        world-1, each rank contributing the one it converted, padded to the longest of the round."""
        import torch.distributed as dist
        lens = [self._segment_frames(n) * net_g.upp - 2 * self.t_pad_tgt for n in seg_samples]
        for k in range(0, len(outs), world):
            ids = list(range(k, min(k + world, len(outs))))
            width = max(lens[i] for i in ids)
            send = torch.zeros(width, device=self.device, dtype=torch.float32)
            mine = k + rank
            if mine < len(outs):
                assert outs[mine].shape[0] == lens[mine], (outs[mine].shape, lens[mine])
                send[:lens[mine]] = outs[mine]
            recv = torch.empty(world * width, device=self.device, dtype=torch.float32)
            dist.all_gather_into_tensor(recv, send, group=self.group)
            recv = recv.view(world, width)
            for i in ids:
                if i != mine:
                    outs[i] = recv[i - k, :lens[i]].clone()

    # ------------------------------------------------------------------ whole utterance
    @staticmethod
    def _reflect_pad(t: torch.Tensor, p: int) -> torch.Tensor:
        """np.pad(t, (p, p), mode="reflect") for a 1-D device tensor."""
        return torch.cat([t[1:p + 1].flip(0), t, t[-p - 1:-1].flip(0)]).contiguous()

    def _cut_points(self, audio64: torch.Tensor):
        """Quiet-point search (vc_infer_pipeline.py:514-528): 160-tap box sum of the reflect-padded signal in fp64 with
        the reference's accumulation order (b200vc_boxsum_f64), then the first argmin of |sum| within +-t_query of every
        t_center multiple."""
        n = audio64.numel()
        opt_ts = []
        if n + self.window > self.t_max:
            audio_pad = self._reflect_pad(audio64, self.window // 2)
            audio_sum = torch.empty(n, dtype=torch.float64, device=audio64.device)
            ops.boxsum_f64(audio_pad, audio_sum, n, self.window)
            centers = list(range(self.t_center, n, self.t_center))
            # first minimum of |sum| in every +-t_query window; ONE device->host copy for all cut points
            rel = torch.stack([torch.argmin(audio_sum[t - self.t_query: t + self.t_query].abs()) for t in centers]).cpu().tolist()
            opt_ts = [t - self.t_query + int(r) for t, r in zip(centers, rel)]
        return opt_ts

    @_ffi.on_device
    def pipeline(self, model, net_g, sid, audio, input_audio_path, times, f0_up_key, f0_method, file_index,
                 index_rate, if_f0, filter_radius, tgt_sr, resample_sr, rms_mix_rate, version, protect,
                 crepe_hop_length, f0_file=None):
        if file_index != "" and os.path.exists(file_index) and index_rate != 0:
            try:
                # the reference re-reads the index on every call (:505-507); the device copy is cached per file version
                key = (file_index, os.path.getmtime(file_index), os.path.getsize(file_index))
                if getattr(self, "_index_cache", (None, None))[0] != key:
                    self._index_cache = (key, read_index(file_index, self.device))
                index = self._index_cache[1]
                big_npy = index._host_vectors            # what reconstruct_n(0, ntotal) returns, without the copy
            except Exception as e:
                # the reference continues without an index on a failed read (:508-510); say so loudly — a silently
                # disabled index changes the timbre of every conversion
                traceback.print_exc()
                import warnings
                warnings.warn(f"b200vc: feature index {file_index!r} could not be loaded ({e}); continuing WITHOUT "
                              f"index retrieval (index_rate={index_rate} ignored)", RuntimeWarning)
                index = big_npy = None
        else:
            index = big_npy = None
        dev = self.device
        if isinstance(audio, torch.Tensor):
            a32 = audio.detach().to(dev).float().contiguous()
        else:
            a32 = torch.from_numpy(np.ascontiguousarray(audio, dtype=np.float32)).to(dev)
        if self.exact_hpf:
            audio = torch.from_numpy(np.ascontiguousarray(signal.filtfilt(bh, ah, a32.cpu().numpy()))).to(dev)
        else:
            audio = ops.filtfilt(a32, bh, ah)                      # fp64 on the device (sos cascade)
        opt_ts = self._cut_points(audio)
        s = 0
        audio_opt = []
        t = None
        t1 = ttime()
        audio_pad = self._reflect_pad(audio, self.t_pad)
        p_len = audio_pad.shape[0] // self.window
        inp_f0 = None
        if hasattr(f0_file, "name"):
            try:
                with open(f0_file.name, "r") as f:
                    lines = f.read().strip("\n").split("\n")
                inp_f0 = np.array([[float(i) for i in line.split(",")] for line in lines], dtype="float32")
            except Exception:
                traceback.print_exc()
        sid = torch.tensor(sid, device=self.device).unsqueeze(0).long()
        pitch, pitchf = None, None
        world, rank = 1, 0
        if self.group is not None:
            import torch.distributed as dist
            world, rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        # the padded utterance goes to HBM once; segments are device slices of it
        pad_dev = audio_pad.float()
        w = self.window
        # segment list exactly as the reference walks it (:548-603): (sample range of the padded utterance, F0 frame range)
        segs = []
        for t in opt_ts:
            t = t // w * w
            segs.append((s, t + self.t_pad2 + w, s // w, (t + self.t_pad2) // w))
            s = t
        segs.append((t if t is not None else 0, None, t // w if t is not None else 0, None))
        mine = [i for i in range(len(segs)) if i % world == rank]      # the others: another rank of the group converts them
        # (single-GPU schedule; in a sharded run the ranks keep the validated order: F0 on rank 0 -> broadcast -> segments)
        overlap = (F0_OVERLAP and world == 1 and if_f0 == 1 and f0_method == "rmvpe"
                   and hasattr(getattr(self, "model_rmvpe", None), "infer_from_audio_begin"))
        halves = {}
        pending = None
        if overlap:
            # F0 (rank 0) goes to a side stream; meanwhile the main stream runs the F0-independent half of every segment
            main = torch.cuda.current_stream()
            if rank == 0:
                if getattr(self, "_f0_stream", None) is None:
                    self._f0_stream = torch.cuda.Stream(device=self.device)
                self._f0_stream.wait_stream(main)
                with torch.cuda.stream(self._f0_stream):
                    pending = self.model_rmvpe.infer_from_audio_begin(audio_pad, thred=0.03)
            for i in mine:
                a0, a1, _, _ = segs[i]
                halves[i] = self._vc_features(model, pad_dev[a0:a1], times, index, big_npy, index_rate, version, protect < 0.5, own=True)
        if if_f0 == 1:
            if rank == 0:       # the F0 is one whole-utterance estimate (bidirectional GRU): group rank 0 computes it ...
                if pending is not None:
                    pitch, pitchf = self._coarse_from_f0(self.model_rmvpe.infer_from_audio_end(pending), f0_up_key, inp_f0)
                    torch.cuda.current_stream().wait_stream(self._f0_stream)     # plan buffers of the F0 net are free again
                else:
                    pitch, pitchf = self.get_f0(input_audio_path, audio_pad, p_len, f0_up_key, f0_method, filter_radius,
                                                crepe_hop_length, inp_f0)
                pitch = torch.tensor(pitch[:p_len], device=self.device).unsqueeze(0).long()
                pitchf = torch.tensor(pitchf[:p_len], device=self.device).unsqueeze(0).float()
            else:
                pitch = torch.empty(1, p_len, device=self.device, dtype=torch.int64)
                pitchf = torch.empty(1, p_len, device=self.device, dtype=torch.float32)
            if world > 1:       # ... and broadcasts pitch / pitchf (~300 KB for 4 minutes)
                src = dist.get_global_rank(self.group, 0)
                dist.broadcast(pitch, src=src, group=self.group)
                dist.broadcast(pitchf, src=src, group=self.group)
        t2 = ttime()
        times[1] += t2 - t1
        audio_opt = [None] * len(segs)
        for i, (a0, a1, p0, p1) in enumerate(segs):
            seg = pad_dev[a0:a1]
            if i % world != rank:
                if self._noise_gen is not None:
                    self._draw_noise(net_g, self._segment_frames(seg.shape[0]), upload=False)
                continue
            pi, pfi = (pitch[:, p0:p1], pitchf[:, p0:p1]) if if_f0 == 1 else (None, None)
            if i in halves:
                out = self._vc_synth(net_g, sid, halves.pop(i), pi, pfi, times, protect)
            else:
                out = self.vc(model, net_g, sid, seg, pi, pfi, times, index, big_npy, index_rate, version, protect)
            audio_opt[i] = out[self.t_pad_tgt: -self.t_pad_tgt].clone()
        if world > 1:
            self._gather_segments(audio_opt, [pad_dev[a0:a1].shape[0] for (a0, a1, _, _) in segs], net_g, world, rank)
        audio_dev = torch.cat(audio_opt).contiguous()
        if self.keep_float:
            self.last_float_output = audio_dev.cpu().numpy()   # pre-RMS-mix float waveform (parity tests)
        if rms_mix_rate != 1:
            # change_rms on the device (the reference does it with librosa/torch on the host, :639-640)
            ops.change_rms(audio, 16000, audio_dev, tgt_sr, rms_mix_rate)
        if resample_sr >= 16000 and tgt_sr != resample_sr:
            raise NotImplementedError("resample_sr != 0 needs librosa.resample; rvc_infer always passes 0 (rvc.py:150)")
        if self.keep_float:
            self.last_float_mixed = audio_dev.cpu().numpy()
        out_i16 = ops.to_int16_peak_guard(audio_dev)
        del pitch, pitchf, sid
        if self.return_device:
            return out_i16                        # CoverEngine: the mix reads the utterance from HBM
        return out_i16.cpu().numpy()              # the single D2H of the converted utterance
