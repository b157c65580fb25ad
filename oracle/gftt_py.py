"""CPU oracle of the GFTT/ORB detector (Kp/DetectorStrategy=8) -- TEST INFRASTRUCTURE ONLY.

rtabmap::GFTT_ORB (corelib/src/Features2d.cpp:2141-2178, :2352-2356) is cv::GFTTDetector::detect followed by cv::ORB::compute, inside the
same Feature2D wrapper as strategy 2 (depth mask, limitKeypoints, 3-D lifting: oracle/feature2d_py.py).  `detect_describe_gftt`
composes those calls with opencv-python 4.13, the dependency itself.

`corner_min_eig` and `select_corners` restate cv::cornerMinEigenVal(gray, 3, 3) and the selection of cv::goodFeaturesToTrack in
numpy, in the arithmetic the CUDA kernels (rtabmap_b200/csrc/gftt.cuh) use; tests/test_oracle_gftt.py pins them bit for bit to cv2:
  * Sobel, scale s = 1/(4*3*255) as a float, reflect-101 border:
      dx = fma(U + D, s, C * 2s), U/C/D = I[x+1] - I[x-1] on the rows above, at and below;
      row pass of column x: r = fma(R, s, fma(M, 2s, L * s)) for x < (w // 32) * 32, ((L * s + M * 2s) + R * s) without fused
      multiply-add in the last w % 32 columns; dy = r[y+1] - r[y-1].  32 is the width in pixels (one v_uint8 register) of OpenCV's
      x86 AVX2 row filter: its vector body fuses, its scalar tail does not.  The pinned target is x86 opencv-python 4.13;
      tests/test_oracle_gftt_edges.py probes the host's cv2 for that boundary (other platforms' vector widths differ);
  * products dx*dx, dx*dy, dy*dy in float; the unnormalised 3x3 box filter sums each row in double, (p[x-1] + p[x]) + p[x+1],
    then keeps a RUNNING column sum in double from the top of the image down (add the row entering, output, subtract the row
    leaving).  The running sum is not exact (the Sobel fma leaves residuals of ~1e-12 whose squares reach below the double's
    range relative to the large terms), so a direct 3x3 sum differs from OpenCV on a few pixels per image;
  * a = 0.5 xx, c = 0.5 yy, lambda = (a + c) - sqrt((a - c)^2 + b^2) in float, without fused multiply-add;
  * threshold = float(max(lambda inside the mask) * quality), kept where lambda > threshold (THRESH_TOZERO); 3x3 dilation; candidates
    are interior pixels with a non-zero value equal to the dilated one, inside the mask; sorted by value descending, the LATER raster
    position first among equals (greaterThanPtr compares the addresses);
  * minDistance >= 1: a grid of cvRound(minDistance) cells, a corner is kept when no kept corner in the 3x3 neighbouring cells lies at a
    squared distance below minDistance^2; minDistance < 1: no filter; stop at maxCorners kept.
"""
from __future__ import annotations

from dataclasses import dataclass

import cv2
import numpy as np

from . import feature2d_py as f2d


@dataclass
class GfttParams:
    quality_level: float = 0.001  # GFTT/QualityLevel
    min_distance: float = 7.0     # GFTT/MinDistance
    block_size: int = 3           # GFTT/BlockSize
    use_harris: bool = False      # GFTT/UseHarrisDetector
    k: float = 0.04               # GFTT/K


def _fma(a, b, c):
    # float fma through double: the product of two floats is exact in double, the sum rounds in double and again to float (a double
    # rounding that could differ from one fused rounding; tests/test_oracle_gftt.py shows it does not on these operands)
    return (a.astype(np.float64) * np.float64(b) + c.astype(np.float64)).astype(np.float32)


SIMD_ROW_WIDTH = 32  # pixels per vector of OpenCV's x86 AVX2 row filter (v_uint8): the columns its fused vector body covers


def corner_min_eig(gray: np.ndarray, simd_width: int = SIMD_ROW_WIDTH) -> np.ndarray:
    """cv::cornerMinEigenVal(gray, 3, 3); the row pass of dy is fused in the first (w // simd_width) * simd_width columns (simd_width=1:
    fused everywhere, the tests' way to see which pixels the unfused tail changes)"""
    f = np.float32
    s = f(1.0 / 3060.0)
    s2 = f(2.0 / 3060.0)
    P = np.pad(gray, 1, mode="reflect").astype(np.float32)
    D = P[:, 2:] - P[:, :-2]
    dx = _fma(D[:-2] + D[2:], s, D[1:-1] * s2)
    h, w = gray.shape
    r = _fma(P[:, 2:], s, _fma(P[:, 1:-1], s2, P[:, :-2] * s))
    x0 = (w // simd_width) * simd_width
    r[:, x0:] = (P[:, x0:w] * s + P[:, x0 + 1:w + 1] * s2) + P[:, x0 + 2:w + 2] * s
    dy = r[2:] - r[:-2]

    def box(p):
        q = np.pad(p, 1, mode="reflect").astype(np.float64)
        rs = (q[:, :-2] + q[:, 1:-1]) + q[:, 2:]
        out = np.empty((h, w), np.float32)
        acc = (np.zeros(w) + rs[0]) + rs[1]
        for y in range(h):
            s0 = acc + rs[y + 2]
            out[y] = s0
            acc = s0 - rs[y]
        return out

    a = box(dx * dx) * f(0.5)
    b = box(dx * dy)
    c = box(dy * dy) * f(0.5)
    t = a - c
    return (a + c) - np.sqrt(t * t + b * b)


def select_corners(eig: np.ndarray, mask, max_corners: int, quality: float, min_distance: float) -> np.ndarray:
    """goodFeaturesToTrack after the corner map: [n, 3] float32 rows (x, y, quality) in OpenCV's order."""
    h, w = eig.shape
    inside = mask != 0 if mask is not None else np.ones((h, w), bool)
    max_val = float(eig[inside].max()) if inside.any() else 0.0
    thr = np.float32(max_val * quality)
    t = np.where(eig > thr, eig, np.float32(0))
    q = np.pad(t, 1, mode="constant", constant_values=-np.inf)
    dil = np.max(np.stack([q[dy:dy + h, dx:dx + w] for dy in range(3) for dx in range(3)]), axis=0)
    cand = (t != 0) & (t == dil) & inside
    cand[0, :] = cand[-1, :] = False
    cand[:, 0] = cand[:, -1] = False
    idx = np.flatnonzero(cand)
    vals = t.ravel()[idx]
    order = np.lexsort((-idx, -vals.astype(np.float64)))  # value descending, then raster index descending
    idx, vals = idx[order], vals[order]
    out = []
    if min_distance >= 1:
        cell = int(np.rint(min_distance))
        gw, gh = (w + cell - 1) // cell, (h + cell - 1) // cell
        grid = [[] for _ in range(gw * gh)]
        md2 = min_distance * min_distance
        for i, v in zip(idx.tolist(), vals.tolist()):
            y, x = divmod(i, w)
            xc, yc = x // cell, y // cell
            good = True
            for yy in range(max(0, yc - 1), min(gh - 1, yc + 1) + 1):
                for xx in range(max(0, xc - 1), min(gw - 1, xc + 1) + 1):
                    for px, py in grid[yy * gw + xx]:
                        if (x - px) ** 2 + (y - py) ** 2 < md2:
                            good = False
                            break
                    if not good:
                        break
                if not good:
                    break
            if good:
                grid[yc * gw + xc].append((x, y))
                out.append((x, y, v))
                if max_corners > 0 and len(out) == max_corners:
                    break
    else:
        for i, v in zip(idx.tolist(), vals.tolist()):
            y, x = divmod(i, w)
            out.append((x, y, v))
            if max_corners > 0 and len(out) == max_corners:
                break
    return np.array(out, np.float32).reshape(-1, 3)


def make_gftt(p: f2d.OrbParams, g: GfttParams):
    return cv2.GFTTDetector_create(p.n_features, g.quality_level, g.min_distance, g.block_size, g.use_harris, g.k)


def detect_describe_gftt(image: np.ndarray, depth, K4, p: f2d.OrbParams = f2d.OrbParams(), g: GfttParams = GfttParams()):
    """GFTT_ORB in Memory::createSignature's feature block: gray -> mask -> GFTTDetector::detect -> limitKeypoints -> ORB::compute ->
    generateKeypoints3D.  Returns (keypoints [n,6] float32 = x,y,size,angle,response,octave; desc [n,32]; xyz [n,3])."""
    gray = cv2.cvtColor(image, cv2.COLOR_BGR2GRAY) if image.ndim == 3 else image
    mask = f2d.depth_mask(depth, p) if (depth is not None and p.depth_as_mask) else None
    kps = make_gftt(p, g).detect(gray, mask)
    kps = f2d.limit_keypoints(kps, p.n_features)
    kps, desc = f2d.make_orb(p).compute(gray, kps)
    if desc is None:
        desc = np.zeros((0, 32), np.uint8)
    xyz = f2d.keypoints_3d(kps, depth, K4, p) if depth is not None else np.full((len(kps), 3), np.nan, np.float32)
    arr = np.array([[k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave] for k in kps], np.float32).reshape(-1, 6)
    return arr, desc, xyz
