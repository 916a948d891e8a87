"""TEST INFRASTRUCTURE ONLY — numpy restatement of the faiss calls on the RVC path.

faiss-cpu 1.7.3 (requirements.txt:3) is a third-party dependency absent from the reference repository: the
`added_IVF{n}_Flat_nprobe_1_*.index` files (rvc_models/MODELS.txt, README.md:165) are IndexIVFFlat / L2 /
nprobe=1, restated from the published algorithm; PARITY UNPINNED against real faiss (tie order in
particular).  Call sites: vc_infer_pipeline.py:505-507 (read_index, reconstruct_n), :421 (search k=8).
"""
from __future__ import annotations

import numpy as np


class IvfFlatIndex:
    """IndexIVFFlat(d, nlist, METRIC_L2) with nprobe=1 after train()+add(): vectors keep insertion ids."""

    def __init__(self, centroids: np.ndarray, vectors: np.ndarray):
        self.centroids = np.ascontiguousarray(centroids, dtype=np.float32)
        self.vectors = np.ascontiguousarray(vectors, dtype=np.float32)
        self.ntotal = self.vectors.shape[0]
        self.d = self.vectors.shape[1]
        self.assign = self._nearest_centroid(self.vectors)
        self.lists = [np.nonzero(self.assign == c)[0] for c in range(self.centroids.shape[0])]

    def _nearest_centroid(self, x: np.ndarray) -> np.ndarray:
        out = np.empty(len(x), dtype=np.int64)
        c2 = (self.centroids.astype(np.float64) ** 2).sum(1)
        for s in range(0, len(x), 4096):
            xb = x[s:s + 4096].astype(np.float64)
            dist = c2[None, :] - 2.0 * xb @ self.centroids.astype(np.float64).T
            out[s:s + 4096] = dist.argmin(1)
        return out

    def reconstruct_n(self, i0: int, n: int) -> np.ndarray:
        return self.vectors[i0:i0 + n].copy()

    def search(self, x: np.ndarray, k: int = 8):
        x = np.ascontiguousarray(x, dtype=np.float32)
        q_list = self._nearest_centroid(x)
        D = np.full((len(x), k), np.inf, dtype=np.float32)
        I = np.full((len(x), k), -1, dtype=np.int64)
        for t in range(len(x)):
            ids = self.lists[q_list[t]]
            if len(ids) == 0:
                continue
            diff = self.vectors[ids] - x[t][None, :]
            dist = (diff * diff).sum(1, dtype=np.float32)
            order = np.argsort(dist, kind="stable")[:k]
            D[t, :len(order)] = dist[order]
            I[t, :len(order)] = ids[order]
        return D, I


def blend(index: IvfFlatIndex, big_npy: np.ndarray, feats: np.ndarray, index_rate: float) -> np.ndarray:
    """vc_infer_pipeline.py:421-431 on a float32 [T, d] feature matrix."""
    score, ix = index.search(feats, k=8)
    with np.errstate(divide="ignore", invalid="ignore"):
        weight = np.square(1 / score)
        weight /= weight.sum(axis=1, keepdims=True)
    npy = np.sum(big_npy[ix] * np.expand_dims(weight, axis=2), axis=1)
    return (npy * np.float32(index_rate) + np.float32(1 - index_rate) * feats).astype(np.float32)
