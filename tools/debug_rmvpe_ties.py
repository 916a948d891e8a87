"""How often does the coarse pitch of the GPU rmvpe differ from the CPU oracle, and is every difference an fp32
near-tie of the salience argmax?  (random-weight nets have noise-like salience, SURVEY.md §7.3 item 1)"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aicovergen_b200.rmvpe import RMVPEB200  # noqa: E402
from aicovergen_b200.synthetic import make_rmvpe_state_dict  # noqa: E402
from oracle import rmvpe as orm  # noqa: E402

sd = make_rmvpe_state_dict()
net = RMVPEB200(sd, device="cuda:0")
rng = np.random.default_rng(0)
tot = mis = 0
for secs, kind in [(1.0, "sweep"), (2.0, "sweep"), (5.0, "sweep"), (3.0, "noise"), (6.0, "noise"), (4.0, "mix")]:
    n = int(16000 * secs)
    t = np.arange(n) / 16000.0
    sw = 0.5 * np.sin(2 * np.pi * (100 * t + 450 / secs * t * t))
    x = {"sweep": sw, "noise": 0.3 * rng.standard_normal(n), "mix": 0.7 * sw + 0.1 * rng.standard_normal(n)}[kind].astype(np.float32)
    hid = orm.mel2hidden(sd, orm.log_mel(torch.from_numpy(x)[None]))[0].numpy()
    sal = net.salience_from_audio(torch.from_numpy(x).cuda()).cpu().numpy()
    f0_ref = orm.decode(hid.copy(), 0.03)
    f0 = net.infer_from_audio(x, 0.03)
    m = orm.coarse_pitch(f0)[0] != orm.coarse_pitch(f0_ref)[0]
    top2 = np.sort(hid, axis=1)[:, -2:]
    gap = top2[:, 1] - top2[:, 0]
    print(f"{kind} {secs}s: frames {len(f0)} mismatches {int(m.sum())} salience max err {np.abs(sal - hid).max():.2e} "
          f"min gap {gap.min():.2e} gaps at mismatches {np.round(gap[m], 6).tolist()} argmax flips {int((sal.argmax(1) != hid.argmax(1)).sum())}")
    tot += len(f0)
    mis += int(m.sum())
print(f"TOTAL {mis}/{tot}")
