"""GPU parity: HuBERT (extract_features plug point) vs the CPU oracle restatement (oracle/hubert.py,
cross-checked against transformers.HubertModel).  BASELINE.json config 2: 30 s of 16 kHz audio."""
import numpy as np
import pytest
import torch

from aicovergen_b200 import tapgemm as tg
from aicovergen_b200.synthetic import make_hubert_state_dict

pytestmark = pytest.mark.gpu


def signal(seconds, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = int(16000 * seconds)
    t = torch.arange(n) / 16000.0
    dur = n / 16000.0
    sweep = 0.5 * torch.sin(2 * np.pi * (100 * t + 450 / dur * t * t))
    return (0.1 * torch.randn(n, generator=g) + sweep).float()[None]


def rel_rms(a, b):
    return ((a.double() - b.double()).pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt()).item()


@pytest.mark.parametrize("backend,tol", [(tg.BACKEND_SIMT, 5e-5), (tg.BACKEND_TC, 1e-2)])
@pytest.mark.parametrize("seconds,layer", [(1.37, 12), (30.0, 12), (4.0, 9)])
def test_hubert_features_parity(backend, tol, seconds, layer):
    from aicovergen_b200.hubert import HubertB200
    from oracle import hubert as oh

    sd = make_hubert_state_dict()
    x = signal(seconds)
    ref = oh.extract_features(sd, x, layer)
    net = HubertB200(sd, "cuda:0", backend=backend)
    got, _ = net.extract_features(source=x.cuda(), padding_mask=torch.zeros_like(x, dtype=torch.bool).cuda(),
                                  output_layer=layer)
    torch.cuda.synchronize()
    name = "tc" if backend == tg.BACKEND_TC else "simt"
    assert got.shape == ref.shape, (got.shape, ref.shape)
    e = rel_rms(got.cpu(), ref)
    print(f"[hubert {name} {seconds}s L{layer}] T={ref.shape[1]} rel rms err {e:.3e}")
    assert torch.isfinite(got).all()
    assert e < tol
    if layer == 9:
        fp = net.final_proj(got)
        e2 = rel_rms(fp.cpu(), oh.final_proj(sd, ref))
        print(f"[hubert {name}] final_proj rel rms err {e2:.3e}")
        assert e2 < tol * 2
