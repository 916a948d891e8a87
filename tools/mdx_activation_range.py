"""fp16-storage safety probe for the MDX U-Net (CPU, test infrastructure): runs the oracle network on one chunk and records
max |value| of every tensor the GPU plan would STORE in fp16 mode (post-activation conv outputs, the TDF hidden layer after
the s2 scaling, block outputs x + tdf(x), the skip product).  fp16 overflows at 65504; values far below that are safe.
usage: python tools/mdx_activation_range.py [--dim-f 3072 --dim-t 256 --g 48] [--real-stft]"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aicovergen_b200.synthetic import make_mdx_state_dict  # noqa: E402
from oracle import mdx as om  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--dim-f", type=int, default=3072)
ap.add_argument("--dim-t", type=int, default=256)
ap.add_argument("--g", type=int, default=48)
ap.add_argument("--n-fft", type=int, default=7680)
ap.add_argument("--scale", type=float, default=3.0, help="std of the random spectrogram (tests use 3.0)")
ap.add_argument("--real-stft", action="store_true", help="feed the STFT of a full-scale synthetic song chunk instead of noise")
ap.add_argument("--calibrate", action="store_true", help="fit the BatchNorm statistics first (synthetic.calibrate_mdx_batchnorm)")
args = ap.parse_args()

sd = make_mdx_state_dict(dim_f=args.dim_f, dim_t=args.dim_t, g=args.g)
dim_f, dim_t, g, l, n, bn, k, dim_c = [int(v) for v in sd["_meta"]]
if args.real_stft:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    mp = om.MdxParams(dim_f, dim_t, args.n_fft)
    song = torch.from_numpy(bench.synth_song(30.0, 0))
    song = song / song.abs().max()
    x = mp.stft(song[None, :, 44100:44100 + mp.chunk_size])
else:
    x = torch.randn(1, 4, dim_f, dim_t, generator=torch.Generator().manual_seed(1)) * args.scale
if args.calibrate:
    from aicovergen_b200.synthetic import calibrate_mdx_batchnorm
    if args.real_stft:   # calibrate on a chunk of a DIFFERENT synthetic song (seed 1), evaluate on seed 0
        other = torch.from_numpy(bench.synth_song(30.0, 1))
        other = other / other.abs().max()
        calib_in = mp.stft(other[None, :, 2 * 44100:2 * 44100 + mp.chunk_size])
    else:                # a different noise draw of the same scale
        calib_in = torch.randn(1, 4, dim_f, dim_t, generator=torch.Generator().manual_seed(7)) * float(x.std())
    sd = calibrate_mdx_batchnorm(sd, calib_in)
rec = {}


def note(name, t):
    rec[name] = max(rec.get(name, 0.0), float(t.abs().max()))
    return t


def tfc_tdf(p, x):
    for j in range(l):
        x = note(f"{p}.c{j}", F.relu(om._bn(sd, f"{p}.tfc.H.{j}.1", F.conv2d(x, sd[f"{p}.tfc.H.{j}.0.weight"], sd[f"{p}.tfc.H.{j}.0.bias"], padding=1))))
    h = F.relu(om._bn(sd, f"{p}.tdf.1", F.linear(x, sd[f"{p}.tdf.0.weight"])))
    s2 = sd[f"{p}.tdf.4.weight"] / torch.sqrt(sd[f"{p}.tdf.4.running_var"] + om.BN_EPS)
    note(f"{p}.h*s2", h * s2[None, :, None, None])          # what the plan stores: relu(...) * s2
    t = F.relu(om._bn(sd, f"{p}.tdf.4", F.linear(h, sd[f"{p}.tdf.3.weight"])))
    return note(f"{p}.out", x + t)


with torch.no_grad():
    print(f"input spectrogram max |x| = {float(x.abs().max()):.1f}")
    x = note("first", F.relu(om._bn(sd, "first_conv.1", F.conv2d(x, sd["first_conv.0.weight"], sd["first_conv.0.bias"])))).transpose(-1, -2)
    skips = []
    for i in range(n):
        x = tfc_tdf(f"encoding_blocks.{i}", x)
        skips.append(x)
        x = note(f"ds.{i}", F.relu(om._bn(sd, f"ds.{i}.1", F.conv2d(x, sd[f"ds.{i}.0.weight"], sd[f"ds.{i}.0.bias"], stride=2))))
    x = tfc_tdf("bottleneck_block", x)
    for i in range(n):
        x = F.relu(om._bn(sd, f"us.{i}.1", F.conv_transpose2d(x, sd[f"us.{i}.0.weight"], sd[f"us.{i}.0.bias"], stride=2)))
        x = note(f"us.{i}*skip", x * skips[-i - 1])
        x = tfc_tdf(f"decoding_blocks.{i}", x)
worst = max(rec.items(), key=lambda kv: kv[1])
for k_, v in rec.items():
    print(f"{k_:32s} {v:12.2f}")
print(f"\nlargest stored value: {worst[1]:.1f} at {worst[0]}  (fp16 max 65504; headroom x{65504 / worst[1]:.1f})")
