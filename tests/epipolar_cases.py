"""Seeded point sets and signature pairs for the epipolar check tests (test_oracle_epipolar.py, test_gpu_epipolar.py)."""
from __future__ import annotations

import numpy as np

K = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
SIZES = (7, 8, 11, 14, 15, 16, 50, 300, 1000)
OUTLIERS = (0.0, 0.3, 0.5, 0.7)
KINDS = ("general", "plane", "zero", "dup", "line")


def _rot(r):
    th = np.linalg.norm(r)
    if th == 0:
        return np.eye(3)
    k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def point_sets(n: int, outliers: float, kind: str, seed: int, noise: float = 0.3):
    """(p1, p2) float32 [n, 2]: a two-view scene with pixel noise and a share of random outliers.  kind: general (depths 2-8 m),
    plane (a fronto-parallel plane: a homography), zero (no motion), dup (four copies of one point), line (half of the image-1
    points, at least 7, on one line)."""
    rng = np.random.default_rng(seed)
    z = np.full(n, 4.0) if kind == "plane" else rng.uniform(2, 8, n)
    X = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), z], 1)
    R, t = (np.eye(3), np.zeros(3)) if kind == "zero" else (_rot(rng.normal(0, 0.05, 3)), rng.normal(0, 0.3, 3))
    x1 = (K @ X.T).T
    x1 = x1[:, :2] / x1[:, 2:]
    x2 = (K @ ((R @ X.T).T + t).T).T
    x2 = x2[:, :2] / x2[:, 2:]
    x1 += rng.normal(0, noise, x1.shape)
    x2 += rng.normal(0, noise, x2.shape)
    k = int(round(outliers * n))
    idx = rng.choice(n, k, replace=False)
    x2[idx] = rng.uniform([0, 0], [640, 480], (k, 2))
    if kind == "dup":
        x1[1:4] = x1[0]
        x2[1:4] = x2[0]
    if kind == "line":
        m = max(7, n // 2)
        s = rng.uniform(0, 600, m)
        x1[:m] = np.stack([s, 0.3 * s + 20], 1)
    return x1.astype(np.float32), x2.astype(np.float32)


def corpus(max_n: int = 1000):
    """(kind, n, outliers, seed) of the seeded corpus."""
    out = []
    for kind in KINDS:
        for n in SIZES:
            if n > max_n:
                continue
            for o in OUTLIERS:
                for seed in range(2 if n >= 300 else 4):
                    out.append((kind, n, o, 1000 * SIZES.index(n) + 100 * OUTLIERS.index(o) + 10 * KINDS.index(kind) + seed))
    return out


def signature_pair(p1, p2, seed: int, extra: int = 0, dup: int = 0, negative: int = 0):
    """Word ids and keypoints of two signatures whose unique shared words are the rows of p1 / p2 in ascending id order, shuffled into
    the rows, with `extra` words on each side that the other lacks, `dup` ids repeated on one side and `negative` negative ids."""
    rng = np.random.default_rng(seed)
    n = len(p1)
    ids = np.sort(rng.choice(np.arange(0, 10 * (n + extra + dup + 10)), n + 2 * extra + dup, replace=False)).astype(np.int32)
    shared = ids[:n]
    rest = rng.permutation(ids[n:])
    only_a, only_b, dups = rest[:extra], rest[extra:2 * extra], rest[2 * extra:]
    ia = np.concatenate([shared, only_a, dups, dups, -1 - np.arange(negative, dtype=np.int32)])
    ib = np.concatenate([shared, only_b, dups, -1 - np.arange(negative, dtype=np.int32)])
    ua = np.concatenate([p1, rng.uniform(0, 640, (len(ia) - n, 2))]).astype(np.float32)
    ub = np.concatenate([p2, rng.uniform(0, 640, (len(ib) - n, 2))]).astype(np.float32)
    pa, pb = rng.permutation(len(ia)), rng.permutation(len(ib))
    return ia[pa], ua[pa], ib[pb], ub[pb]
