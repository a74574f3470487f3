"""Synthetic match graphs with the shapes of BASELINE.json's configs (SURVEY 8d).

There is no network for the LFE / ETH3D datasets and the two-view network that
produces the real flow grids (two-view-refinement/, out of scope) is not run
here, so the solver is fed synthetic `MatchingFile` content with the same
structure: K keypoints per image observing a pool of 3-D points, mutual-NN
style matches (<= 1 match per keypoint per pair, feature_matchers.py:18,54),
3x3x2 fp32 flow grids sampled at {-0.5, 0, 0.5}^2 in units of 16 px
(refinement.py:83, colmap_utils.py:135-136), plus a fraction of outlier matches
that link unrelated keypoints (these create inter-track Tukey edges and
meta-components larger than #images, exercising solve.cc:311-343).

    d_ab(g) = (t_b - t_a) + B g + eps      sampled around keypoint a
    t ~ U(-0.3, 0.3)^2, B ~ U(-0.1, 0.1)^{2x2}, eps ~ N(0, 0.01^2)

`disp2` of a match carries d_12 and `disp1` carries d_21
(compute_match_graph.py:181-187).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Tuple

import numpy as np

from .matchset import MatchSet

# grid sample coordinates in the [3*i+j] order of refinement.py:83 (indexing='ij')
_GRID = np.array([(gi, gj) for gi in (-0.5, 0.0, 0.5) for gj in (-0.5, 0.0, 0.5)], dtype=np.float64)


@dataclass
class SynthConfig:
    name: str
    n_images: int
    kpts: int
    pairs: str            # 'exhaustive' | 'sequential' | 'ring'
    visibility: float
    match_prob: float = 0.8
    outlier_frac: float = 0.05
    window: int = 0       # sequential / ring: |i - j| <= window are paired
    loop: int = 0         # sequential: extra pairs (i, i + loop)
    n_random: int = 0     # ring: extra random partners per image
    vis_halfwidth: int = 0  # sequential / ring: a point is seen within this many frames of its centre
    seed: int = 0
    outlier_match_ratio: float = 0.0  # > 0: cap a pair's outliers at this fraction of its inlier matches


CONFIGS = {
    # BASELINE.json configs[0..4]
    "cfg1": SynthConfig("cfg1", 3, 200, "exhaustive", 0.9, seed=1001),
    "cfg2": SynthConfig("cfg2", 11, 3000, "exhaustive", 0.7, seed=1002),
    "cfg3": SynthConfig("cfg3", 8, 8000, "exhaustive", 0.7, seed=1003),
    "cfg4": SynthConfig("cfg4", 38, 4000, "sequential", 0.7, window=10, loop=19,
                        vis_halfwidth=8, seed=1004),
    # retrieval pairs share few points, so "5 % of K" outliers would be a third of all
    # matches and glue hundreds of tracks together; cap them at 1/8 of the pair's inliers
    # (the ratio the exhaustive configs have)
    "cfg5": SynthConfig("cfg5", 1000, 2000, "ring", 0.7, match_prob=0.3, window=20,
                        n_random=5, vis_halfwidth=12, seed=1005, outlier_match_ratio=0.125),
    # a small ring scene whose components exceed 96 unknowns (exercises the CTA / PCG tier cheaply)
    "ring60": SynthConfig("ring60", 60, 400, "ring", 0.7, match_prob=0.5, window=8,
                          n_random=2, vis_halfwidth=10, seed=1060),
    "ring200": SynthConfig("ring200", 200, 150, "ring", 0.7, match_prob=0.4, window=12,
                           n_random=3, vis_halfwidth=10, seed=1200, outlier_match_ratio=0.125),
}

ALIASES = {"fountain": "cfg2", "herzjesu": "cfg3", "courtyard": "cfg4", "madrid": "cfg5", "tiny": "cfg1"}


def pair_list(cfg: SynthConfig, rng: np.random.Generator) -> List[Tuple[int, int]]:
    n = cfg.n_images
    if cfg.pairs == "exhaustive":  # utils/create_exhaustive_matching_list.py:35-37
        return [(a, b) for a in range(n) for b in range(a + 1, n)]
    if cfg.pairs == "sequential":  # utils/create_sequential_matching_list.py:39-47 (+ loop closures)
        out = [(a, b) for a in range(n) for b in range(a + 1, min(n, a + cfg.window + 1))]
        if cfg.loop:
            seen = set(out)
            for a in range(n - cfg.loop):
                if (a, a + cfg.loop) not in seen:
                    out.append((a, a + cfg.loop))
        return out
    if cfg.pairs == "ring":  # retrieval-style: nearest on a ring + a few random partners (README.md:173)
        seen = set()
        out = []
        for a in range(n):
            for d in range(1, cfg.window + 1):
                b = (a + d) % n
                key = (min(a, b), max(a, b))
                if key not in seen:
                    seen.add(key)
                    out.append(key)
        for a in range(n):
            for b in rng.integers(0, n, size=cfg.n_random).tolist():
                key = (min(a, b), max(a, b))
                if a != b and key not in seen:
                    seen.add(key)
                    out.append(key)
        return out
    raise ValueError(cfg.pairs)


def generate(cfg, scale: float = 1.0, seed: int | None = None, pairs=None) -> MatchSet:
    """Build the MatchSet of a config (name, alias or SynthConfig).  `scale`
    multiplies keypoints per image (for quick tests).  `pairs` ([(a, b)], a != b) replaces the
    config's pair list."""
    if isinstance(cfg, str):
        cfg = CONFIGS[ALIASES.get(cfg, cfg)]
    rng = np.random.default_rng(cfg.seed if seed is None else seed)
    n, K = cfg.n_images, max(2, int(round(cfg.kpts * scale)))
    # --- which 3-D points each image observes --------------------------------
    if cfg.pairs == "exhaustive":
        P = int(round(K / cfg.visibility))
        obs = [np.sort(rng.choice(P, size=K, replace=False)) for _ in range(n)]
    else:
        span = 2 * cfg.vis_halfwidth + 1
        P = int(round(K / cfg.visibility * n / span))
        centre = rng.uniform(0, n, size=P)
        obs = []
        for i in range(n):
            d = np.abs(centre - i)
            if cfg.pairs == "ring":
                d = np.minimum(d, n - d)
            elig = np.nonzero(d <= cfg.vis_halfwidth + 0.5)[0]
            take = min(K, elig.shape[0])
            obs.append(np.sort(rng.choice(elig, size=take, replace=False)))
    # feature index of each observation = random permutation per image
    feat = [rng.permutation(o.shape[0]).astype(np.uint32) for o in obs]
    # keypoint localisation error of each observation, units of 16 px
    terr = [rng.uniform(-0.3, 0.3, size=(o.shape[0], 2)) for o in obs]

    pairs = pair_list(cfg, rng) if pairs is None else [(int(a), int(b)) for a, b in pairs]
    f1s, f2s, sims, d1s, d2s, ptr = [], [], [], [], [], [0]
    n_out = int(round(cfg.outlier_frac * K))
    for (a, b) in pairs:
        _, ia, ib = np.intersect1d(obs[a], obs[b], assume_unique=True, return_indices=True)
        keep = rng.random(ia.shape[0]) < cfg.match_prob
        ia, ib = ia[keep], ib[keep]
        m = ia.shape[0]
        sim = rng.uniform(0.80, 0.99, size=m)
        dt = terr[b][ib] - terr[a][ia]                      # t_b - t_a
        B12 = rng.uniform(-0.1, 0.1, size=(m, 2, 2))
        B21 = rng.uniform(-0.1, 0.1, size=(m, 2, 2))
        d12 = dt[:, None, :] + np.einsum("mkl,gl->mgk", B12, _GRID) + rng.normal(0, 0.01, size=(m, 9, 2))
        d21 = -dt[:, None, :] + np.einsum("mkl,gl->mgk", B21, _GRID) + rng.normal(0, 0.01, size=(m, 9, 2))
        # outliers: unrelated keypoints not yet matched in this pair (mutual-NN => <= 1 match per keypoint)
        free_a = np.setdiff1d(np.arange(obs[a].shape[0]), ia, assume_unique=False)
        free_b = np.setdiff1d(np.arange(obs[b].shape[0]), ib, assume_unique=False)
        k = min(n_out, free_a.shape[0], free_b.shape[0])
        if cfg.outlier_match_ratio > 0:
            k = min(k, int(round(cfg.outlier_match_ratio * m)))
        if k > 0:
            oa = rng.choice(free_a, size=k, replace=False)
            ob = rng.choice(free_b, size=k, replace=False)
            ia = np.concatenate([ia, oa])
            ib = np.concatenate([ib, ob])
            sim = np.concatenate([sim, rng.uniform(0.80, 0.90, size=k)])
            d12 = np.concatenate([d12, rng.uniform(-0.5, 0.5, size=(k, 9, 2))])
            d21 = np.concatenate([d21, rng.uniform(-0.5, 0.5, size=(k, 9, 2))])
        # the matcher emits matches in keypoint order of image 1
        order = np.argsort(feat[a][ia], kind="stable")
        f1s.append(feat[a][ia][order])
        f2s.append(feat[b][ib][order])
        sims.append(sim[order].astype(np.float32))
        d1s.append(d21[order].reshape(-1, 18).astype(np.float32))   # disp1 = grid_displacements21
        d2s.append(d12[order].reshape(-1, 18).astype(np.float32))   # disp2 = grid_displacements12
        ptr.append(ptr[-1] + ia.shape[0])

    cat = lambda xs, dt, shape: (np.concatenate(xs).astype(dt) if xs else np.zeros(shape, dtype=dt))
    ms = MatchSet(
        image_names=["%04d.png" % i for i in range(n)],
        pair_img1=np.array([p[0] for p in pairs], dtype=np.int64),
        pair_img2=np.array([p[1] for p in pairs], dtype=np.int64),
        pair_fact1=np.ones(len(pairs), dtype=np.float32),
        pair_fact2=np.ones(len(pairs), dtype=np.float32),
        pair_ptr=np.array(ptr, dtype=np.int64),
        feat1=cat(f1s, np.uint32, (0,)), feat2=cat(f2s, np.uint32, (0,)),
        sim=cat(sims, np.float32, (0,)),
        disp1=cat(d1s, np.float32, (0, 18)), disp2=cat(d2s, np.float32, (0, 18)),
        meta={"config": cfg.name, "n_images": n, "kpts": K, "seed": cfg.seed if seed is None else seed,
              "scale": scale},
    )
    ms.validate()
    return ms
