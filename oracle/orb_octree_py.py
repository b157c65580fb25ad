"""CPU oracle of the ORB-OCTREE detector (Kp/DetectorStrategy=10) -- TEST INFRASTRUCTURE ONLY.

rtabmap::ORBOctree (corelib/src/Features2d.cpp:2479-2566) wraps the ORB-SLAM2 extractor RTAB-Map ships as its own code
(corelib/src/opencv/ORBextractor.cc).  This module restates it step by step; its primitives are OpenCV's own (opencv-python 4.13):
  tables        constructor, ORBextractor.cc:416-477: float scale chain, float per-level counts, umax
  pyramid       ComputePyramid, :1114-1139: level l = cv2.resize(level l-1, cvRound(cols / s_l) x cvRound(rows / s_l), INTER_LINEAR)
  FAST          ComputeKeyPointsOctTree, :772-855: cv2 FAST (9/16, non-max suppression) on each cell's view, FAST/MinThreshold when
                FAST/Threshold finds nothing
  quadtree      DistributeOctTree, :546-770, with the tie rule below
  angle         IC_Angle, :83-110 (cv2.fastAtan2), on the unblurred level
  blur          GaussianBlur(7x7, sigma 2, REFLECT_101) on a contiguous copy (OpenCV's 8-bit fixed-point path), :1092-1093
  descriptor    computeOrbDescriptor, :114-153, cos/sin of a float angle = the host libm's cosf/sinf (through ctypes)
  output        operator(), :1066-1111: levels in order, pt *= scale for level > 0, size = (int)(31 * scale), octave = level
  wrapper       Features2d.cpp:2515-2556: keypoints whose level-0 mask byte at the truncated coordinates is 0 are dropped, then
                Feature2D::limitKeypoints (oracle/feature2d_py.py), then generateKeypoints3D.

Tie rule.  Phase 2 of DistributeOctTree sorts (size, ExtractorNode*) pairs: among nodes of equal size the order is the order of their heap
addresses, which the reference does not define.  This restatement (and the CUDA kernel) takes the node created later as the larger pointer,
so among equal sizes the latest-created node divides first.  `distribute(..., ties)` records each phase-2 round where that order matters:
"set" when the round stops at N inside a run of equal sizes (where it stops, and so which nodes divide, depends on the heap), "order"
when two divided nodes have the same size (where their children go in the list depends on it).  A level without either event keeps the same keypoints in
the same order under every order of equal-size nodes (each round then divides the same nodes whatever that order); a level with "order"
events only keeps the same set.  `detect_describe_octree(..., tie_report=...)` gives that status per level: None, "order" or "set".

`ref_tables` and `ref_distribute` call the reference's own ORBextractor.cc, compiled against OpenCV stand-ins (orbx.mk ->
_ref/libref_orbx.so); tests/test_oracle_orb_octree.py compares the restatement's tables and quadtree with them.

`kernel_resize` and `kernel_blur` restate the integer arithmetic of the CUDA kernels (rtabmap_b200/csrc/orb_octree.cuh);
tests/test_oracle_orb_octree.py pins them to cv2.resize and cv2.GaussianBlur.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math
import re
from dataclasses import dataclass
from pathlib import Path

import cv2
import numpy as np

from . import feature2d_py as f2d

f32 = np.float32
MAX_LEVELS = 8
CELL = f32(30.0)  # W in ComputeKeyPointsOctTree


@dataclass
class OctreeParams:
    n_features: int = 500        # Kp/MaxFeatures
    n_levels: int = 3            # ORB/NLevels
    scale_factor: float = 2.0    # ORB/ScaleFactor
    edge_threshold: int = 19     # ORB/EdgeThreshold
    fast_threshold: int = 20     # FAST/Threshold (the initial threshold)
    fast_min_threshold: int = 7  # FAST/MinThreshold
    patch_size: int = 31         # ORB/PatchSize
    min_depth: float = 0.0       # Kp/MinDepth
    max_depth: float = 0.0       # Kp/MaxDepth
    depth_as_mask: bool = True   # Mem/DepthAsMask

    def orb(self) -> f2d.OrbParams:
        return f2d.OrbParams(self.n_features, self.n_levels, self.scale_factor, self.edge_threshold, self.fast_threshold, self.patch_size,
                             self.min_depth, self.max_depth, self.depth_as_mask)


HERE = Path(__file__).resolve().parent
REF_ORBX_LIB = HERE / "_ref" / "libref_orbx.so"
_ref_orbx = None


def build() -> None:
    """Compile _ref/libref_orbx.so from the reference's ORBextractor.cc when it is missing and the reference is present."""
    from . import oracle_py as orc

    if not REF_ORBX_LIB.exists() and orc._reference_present():
        import subprocess

        subprocess.run(["make", "-C", str(HERE), "-f", "orbx.mk"], check=True, capture_output=True)


def ref_orbx_lib():
    """The reference's compiled ORBextractor (constructor tables, DistributeOctTree), or None when it has not been built."""
    global _ref_orbx
    if _ref_orbx is None:
        build()
        if not REF_ORBX_LIB.exists():
            return None
        R = ctypes.CDLL(str(REF_ORBX_LIB))
        P, I = ctypes.c_void_p, ctypes.c_int
        R.ref_orbx_tables.argtypes = [I, ctypes.c_float, I, I, P, P, P, P]
        R.ref_orbx_distribute.argtypes = [P, I, I, I, I, P, I]
        _ref_orbx = R
    return _ref_orbx


def ref_tables(n_features: int, scale_factor: float, n_levels: int, patch_size: int = 31):
    """The compiled reference constructor's (mvScaleFactor, mvInvScaleFactor, mnFeaturesPerLevel, umax)."""
    scale = np.zeros(n_levels, np.float32)
    inv = np.zeros(n_levels, np.float32)
    per = np.zeros(n_levels, np.int32)
    umax = np.zeros(patch_size // 2 + 1, np.int32)
    rc = ref_orbx_lib().ref_orbx_tables(n_features, float(scale_factor), n_levels, patch_size, *[a.ctypes.data_as(ctypes.c_void_p) for a in
                                                                                              (scale, inv, per, umax)])
    assert rc == 0
    return list(scale), list(inv), per.tolist(), umax.tolist()


def ref_distribute(keys, w: int, h: int, n: int) -> list[int]:
    """The compiled reference's DistributeOctTree on the same keys as `distribute`: indices in list order."""
    k = np.array(keys, np.float32).reshape(-1, 3)
    out = np.zeros(max(len(keys), 1), np.int32)
    m = ref_orbx_lib().ref_orbx_distribute(k.ctypes.data_as(ctypes.c_void_p), len(keys), w, h, n, out.ctypes.data_as(ctypes.c_void_p), len(out))
    assert m >= 0
    return out[:m].tolist()


_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.cosf.restype = _libm.sinf.restype = ctypes.c_float
_libm.cosf.argtypes = _libm.sinf.argtypes = [ctypes.c_float]


def cosf(x) -> np.float32:
    return f32(_libm.cosf(float(x)))


def sinf(x) -> np.float32:
    return f32(_libm.sinf(float(x)))


def _pattern() -> np.ndarray:
    src = (Path(__file__).resolve().parent.parent / "rtabmap_b200" / "csrc" / "orb_pattern.h").read_text()
    body = src[src.index("= {") + 3:src.index("};")]
    return np.array([int(v) for v in re.findall(r"-?\d+", body)], np.int32).reshape(256, 4)


PATTERN = _pattern()


def _round_half_even(v) -> int:
    return int(np.rint(v))


def roundf(v) -> int:
    """std::round of a float: halves away from zero."""
    v = float(v)
    r = math.floor(abs(v) + 0.5) if abs(v) - math.floor(abs(v)) >= 0.5 else math.floor(abs(v))
    return int(math.copysign(r, v))


def tables(n_features: int, scale_factor: float, n_levels: int, patch_size: int = 31):
    """(mvScaleFactor, mvInvScaleFactor, mnFeaturesPerLevel, umax) as the ORBextractor constructor computes them."""
    sf = f32(scale_factor)
    scale = [f32(1.0)]
    for _ in range(1, n_levels):
        scale.append(f32(scale[-1] * sf))
    inv = [f32(f32(1.0) / s) for s in scale]
    factor = f32(f32(1.0) / sf)
    nd = f32(f32(f32(n_features) * f32(f32(1) - factor)) / f32(f32(1) - f32(math.pow(float(factor), float(n_levels)))))
    per, total = [], 0
    for _ in range(n_levels - 1):
        per.append(_round_half_even(nd))
        total += per[-1]
        nd = f32(nd * factor)
    per.append(max(n_features - total, 0))
    half = patch_size // 2
    vmax = math.floor(f32(f32(f32(half) * f32(math.sqrt(2.0))) / f32(2)) + f32(1))
    vmin = math.ceil(f32(f32(f32(half) * f32(math.sqrt(2.0))) / f32(2)))
    umax = [0] * (half + 1)
    for v in range(vmax + 1):
        umax[v] = _round_half_even(math.sqrt(float(half * half) - v * v))
    v0 = 0
    for v in range(half, vmin - 1, -1):
        while umax[v0] == umax[v0 + 1]:
            v0 += 1
        umax[v] = v0
        v0 += 1
    return scale, inv, per, umax


def level_sizes(width: int, height: int, inv) -> list[tuple[int, int]]:
    return [(_round_half_even(f32(f32(width) * s)), _round_half_even(f32(f32(height) * s))) for s in inv]


def check_params(width: int, height: int, p: OctreeParams) -> str | None:
    """The message of the inputs the engine refuses (LCD_ERR_INVALID), or None: the reference divides by zero, indexes out of range or
    reads outside the blurred level on them."""
    if not (1 <= p.n_levels <= MAX_LEVELS):
        return "ORB/NLevels"
    if not (math.isfinite(p.scale_factor) and p.scale_factor > 1.0):
        return "ORB/ScaleFactor"
    if p.patch_size != 31:
        return "ORB/PatchSize"
    if p.edge_threshold < 19:
        return "ORB/EdgeThreshold"
    if not (0 <= p.fast_threshold <= 255) or not (0 <= p.fast_min_threshold <= 255):
        return "FAST threshold"
    if p.n_features <= 0:
        return "Kp/MaxFeatures"
    _, inv, _, _ = tables(p.n_features, p.scale_factor, p.n_levels)
    for (w, h) in level_sizes(width, height, inv):
        bw, bh = w - 2 * (p.edge_threshold - 3), h - 2 * (p.edge_threshold - 3)
        if bw < 30 or bh < 30:
            return "level span"
        if roundf(f32(bw) / f32(bh)) == 0:
            return "level aspect"
    return None


def cell_grid(w: int, h: int, edge: int):
    """The cells of ComputeKeyPointsOctTree on a w x h level: [(i, j, y0, y1, x0, x1)] in row-major order, plus (wCell, hCell)."""
    min_b = edge - 3
    max_bx, max_by = w - edge + 3, h - edge + 3
    width, height = f32(max_bx - min_b), f32(max_by - min_b)
    n_cols, n_rows = int(f32(width / CELL)), int(f32(height / CELL))
    w_cell = int(math.ceil(f32(width / f32(n_cols))))
    h_cell = int(math.ceil(f32(height / f32(n_rows))))
    cells = []
    for i in range(n_rows):
        ini_y = f32(min_b + i * h_cell)
        max_y = f32(ini_y + f32(h_cell + 6))
        if ini_y >= f32(max_by - 3):
            continue
        if max_y > f32(max_by):
            max_y = f32(max_by)
        for j in range(n_cols):
            ini_x = f32(min_b + j * w_cell)
            max_x = f32(ini_x + f32(w_cell + 6))
            if ini_x >= f32(max_bx - 6):
                continue
            if max_x > f32(max_bx):
                max_x = f32(max_bx)
            cells.append((i, j, int(ini_y), int(max_y), int(ini_x), int(max_x)))
    return cells, w_cell, h_cell


def fast_cells(level: np.ndarray, edge: int, thr: int, min_thr: int):
    """Keys to distribute: [(x, y, response)] relative to (edge - 3, edge - 3), cells in row-major order, raster order in a cell."""
    cells, w_cell, h_cell = cell_grid(level.shape[1], level.shape[0], edge)
    fast_ini = cv2.FastFeatureDetector_create(thr, True)
    fast_min = cv2.FastFeatureDetector_create(min_thr, True)
    keys = []
    for (i, j, y0, y1, x0, x1) in cells:
        view = np.ascontiguousarray(level[y0:y1, x0:x1])
        kps = fast_ini.detect(view)
        if not kps:
            kps = fast_min.detect(view)
        for k in kps:
            keys.append((int(k.pt[0]) + j * w_cell, int(k.pt[1]) + i * h_cell, float(k.response)))
    return keys


class _Node:
    __slots__ = ("x0", "y0", "x1", "y1", "keys", "no_more", "rank")

    def __init__(self, x0, y0, x1, y1, keys, rank):
        self.x0, self.y0, self.x1, self.y1, self.keys, self.rank = x0, y0, x1, y1, keys, rank
        self.no_more = len(keys) == 1


def _divide(n: _Node, keys):
    hx = (n.x1 - n.x0 + 1) // 2  # ceil(float(UR.x - UL.x) / 2) of non-negative integers
    hy = (n.y1 - n.y0 + 1) // 2
    mx, my = n.x0 + hx, n.y0 + hy
    parts = ([], [], [], [])
    for k in n.keys:
        x, y = keys[k][0], keys[k][1]
        parts[(0 if y < my else 2) + (0 if x < mx else 1)].append(k)
    rect = ((n.x0, n.y0, mx, my), (mx, n.y0, n.x1, my), (n.x0, my, mx, n.y1), (mx, my, n.x1, n.y1))
    return [(rect[c], parts[c]) for c in range(4)]


def distribute(keys, w: int, h: int, n: int, ties: list | None = None):
    """DistributeOctTree on keys relative to the level's border (width w = maxX - minX, height h): indices into keys, in list order."""
    n_ini = roundf(f32(w) / f32(h))
    hx = f32(f32(w) / f32(n_ini))
    ini = [_Node(int(f32(hx * f32(i))), 0, int(f32(hx * f32(i + 1))), h, [], i) for i in range(n_ini)]
    for idx, k in enumerate(keys):
        ini[int(f32(f32(k[0]) / hx))].keys.append(idx)
    for node in ini:
        node.no_more = len(node.keys) == 1
    lst = [node for node in ini if node.keys]
    rank = n_ini

    def split(node, front, expand):
        nonlocal rank
        for (x0, y0, x1, y1), ks in _divide(node, keys):
            if ks:
                child = _Node(x0, y0, x1, y1, ks, rank)
                rank += 1
                front.append(child)  # push_front: the list starts with the LAST child pushed
                if len(ks) > 1:
                    expand.append(child)

    expand: list = []
    while True:
        prev = len(lst)
        front, rest, expand = [], [], []
        for node in lst:
            if node.no_more:
                rest.append(node)
            else:
                split(node, front, expand)
        lst = front[::-1] + rest
        if len(lst) >= n or len(lst) == prev:
            break
        if len(lst) + 3 * len(expand) > n:
            while True:
                prev = len(lst)
                order = sorted(expand, key=lambda nd: (len(nd.keys), nd.rank))
                expand = []
                front, gone = [], set()
                size = len(lst)
                divided = 0
                for node in reversed(order):
                    before = len(front)
                    split(node, front, expand)
                    gone.add(id(node))
                    divided += 1
                    size += len(front) - before - 1
                    if size >= n:
                        break
                if ties is not None:
                    desc = [len(nd.keys) for nd in reversed(order)]
                    if size >= n and desc.count(desc[divided - 1]) > 1:
                        # the break fell in a run of equal sizes: where it falls, and so which nodes divide, depends on the heap's order
                        ties.append("set")
                    elif len(set(desc[:divided])) < divided:
                        ties.append("order")  # equal sizes among the divided: their children's place in the list is the heap's choice
                lst = front[::-1] + [nd for nd in lst if id(nd) not in gone]
                if len(lst) >= n or len(lst) == prev:
                    break
            break
    out = []
    for node in lst:
        best = node.keys[0]
        for k in node.keys[1:]:
            if keys[k][2] > keys[best][2]:
                best = k
        out.append(best)
    return out


def fast_atan2(y: float, x: float) -> np.float32:
    return f32(cv2.fastAtan2(float(f32(y)), float(f32(x))))


def ic_angle(img: np.ndarray, x: int, y: int, umax, half: int = 15) -> np.float32:
    m01 = m10 = 0
    m10 = int(sum(u * int(img[y, x + u]) for u in range(-half, half + 1)))
    for v in range(1, half + 1):
        d = umax[v]
        row_p = img[y + v, x - d:x + d + 1].astype(np.int64)
        row_m = img[y - v, x - d:x + d + 1].astype(np.int64)
        u = np.arange(-d, d + 1)
        m01 += v * int((row_p - row_m).sum())
        m10 += int((u * (row_p + row_m)).sum())
    return fast_atan2(m01, m10)


FACTOR_PI = f32(math.pi / 180.0)  # (float)(CV_PI / 180.f)


def describe(blurred: np.ndarray, x: int, y: int, angle: np.float32) -> np.ndarray:
    a_ = f32(angle * FACTOR_PI)
    a, b = cosf(a_), sinf(a_)
    px, py = PATTERN[:, [0, 2]].astype(np.float32), PATTERN[:, [1, 3]].astype(np.float32)
    # cvRound(x*b + y*a) rows, cvRound(x*a - y*b) columns: separate float products and sum (no FMA), round half to even
    rows = np.rint((px * b).astype(np.float32) + (py * a).astype(np.float32)).astype(np.int64)
    cols = np.rint((px * a).astype(np.float32) - (py * b).astype(np.float32)).astype(np.int64)
    vals = blurred[y + rows, x + cols].astype(np.int32)
    bits = (vals[:, 0] < vals[:, 1]).astype(np.uint8).reshape(32, 8)
    return (bits << np.arange(8, dtype=np.uint8)).sum(axis=1).astype(np.uint8)


def kernel_resize(src: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """cv2.resize(src, (dw, dh), INTER_LINEAR) for 8-bit images, as orb_oct_resize_kernel computes it: the 2x2 mean at an exact factor
    of 2, otherwise 11-bit fixed-point coefficients, a horizontal pass in int, a vertical pass (b0 * (S0 >> 4)) >> 16 + (b1 * (S1 >> 4))
    >> 16, then (v + 2) >> 2 saturated."""
    sh, sw = src.shape
    s = src.astype(np.int64)
    if sw == 2 * dw and sh == 2 * dh:
        return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)

    def coef(n, n_src):
        scale = 1.0 / (n / n_src)
        f = ((np.arange(n) + 0.5) * scale - 0.5).astype(np.float32)
        i = np.floor(f).astype(np.int64)
        f = (f - i.astype(np.float32)).astype(np.float32)
        f = np.where(i < 0, f32(0), f)
        i = np.maximum(i, 0)
        f = np.where(i >= n_src - 1, f32(0), f)
        i = np.minimum(i, n_src - 1)
        return i, np.rint((f32(1) - f) * f32(2048)).astype(np.int64), np.rint(f * f32(2048)).astype(np.int64)

    xi, xa0, xa1 = coef(dw, sw)
    yi, ya0, ya1 = coef(dh, sh)
    hor = s[:, xi] * xa0 + s[:, np.minimum(xi + 1, sw - 1)] * xa1
    v = ((ya0[:, None] * (hor[yi] >> 4)) >> 16) + ((ya1[:, None] * (hor[np.minimum(yi + 1, sh - 1)] >> 4)) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


GAUSS7_Q8 = (18, 34, 48, 56, 48, 34, 18)  # cv::GaussianBlur's 8-bit fixed-point kernel for 7 taps, sigma 2 (sums to 256)


def kernel_blur(img: np.ndarray) -> np.ndarray:
    """cv2.GaussianBlur(contiguous 8-bit img, (7, 7), 2, 2, BORDER_REFLECT_101), as orb_oct_blur_kernel computes it."""
    k = np.array(GAUSS7_Q8, np.int64)
    h, w = img.shape
    p = np.pad(img.astype(np.int64), 3, mode="reflect")
    row = sum(k[i] * p[:, i:i + w] for i in range(7))
    col = sum(k[i] * row[i:i + h] for i in range(7))
    return np.clip((col + 32768) >> 16, 0, 255).astype(np.uint8)


def extract(gray: np.ndarray, p: OctreeParams, ties: list | None = None):
    """ORBextractor::operator() on a gray image: keypoints [n, 6] float32 (x, y, size, angle, response, octave) and descriptors."""
    scale, inv, per, umax = tables(p.n_features, p.scale_factor, p.n_levels, p.patch_size)
    sizes = level_sizes(gray.shape[1], gray.shape[0], inv)
    levels = [np.ascontiguousarray(gray)]
    for lv in range(1, p.n_levels):
        levels.append(cv2.resize(levels[-1], sizes[lv], interpolation=cv2.INTER_LINEAR))
    edge, min_b = p.edge_threshold, p.edge_threshold - 3
    rows, descs = [], []
    for lv, img in enumerate(levels):
        h, w = img.shape
        keys = fast_cells(img, edge, p.fast_threshold, p.fast_min_threshold)
        bw, bh = (w - edge + 3) - min_b, (h - edge + 3) - min_b
        events: list = []
        sel = distribute(keys, bw, bh, per[lv], events)
        if ties is not None:
            ties.append("set" if "set" in events else ("order" if events else None))
        if not sel:
            continue
        blurred = cv2.GaussianBlur(img.copy(), (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101)
        size = f32(int(f32(f32(p.patch_size) * scale[lv])))
        for k in sel:
            x, y, resp = keys[k][0] + min_b, keys[k][1] + min_b, keys[k][2]
            angle = ic_angle(img, x, y, umax, p.patch_size // 2)
            descs.append(describe(blurred, x, y, angle))
            fx, fy = f32(x), f32(y)
            if lv:
                fx, fy = f32(fx * scale[lv]), f32(fy * scale[lv])
            rows.append((fx, fy, size, angle, f32(resp), f32(lv)))
    kp = np.array(rows, np.float32).reshape(-1, 6)
    desc = np.array(descs, np.uint8).reshape(-1, 32)
    return kp, desc


def detect_describe_octree(image: np.ndarray, depth, K4, p: OctreeParams = OctreeParams(), depth_is_mask: bool = False,
                           tie_report: list | None = None):
    """ORBOctree in Memory::createSignature's feature block: gray -> ORBextractor -> level-0 mask at truncated coordinates ->
    limitKeypoints -> generateKeypoints3D.  Returns (keypoints [n,6] float32; desc [n,32]; xyz [n,3])."""
    gray = cv2.cvtColor(image, cv2.COLOR_BGR2GRAY) if image.ndim == 3 else image
    kp, desc = extract(gray, p, ties=tie_report)
    mask = None
    if depth is not None:
        mask = np.where(depth != 0, 255, 0).astype(np.uint8) if depth_is_mask else (f2d.depth_mask(depth, p.orb()) if p.depth_as_mask else None)
    if mask is not None and len(kp):
        keep = mask[kp[:, 1].astype(np.int64), kp[:, 0].astype(np.int64)] != 0
        kp, desc = kp[keep], desc[keep]
    if p.n_features > 0 and len(kp) > p.n_features:
        order = sorted(range(len(kp)), key=lambda i: (abs(float(kp[i, 4])), i), reverse=True)[:p.n_features]
        kp, desc = kp[order], desc[order]
    if depth is not None and not depth_is_mask:
        kps = [cv2.KeyPoint(float(r[0]), float(r[1]), float(r[2])) for r in kp]
        xyz = f2d.keypoints_3d(kps, depth, K4, p.orb())
    else:
        xyz = np.full((len(kp), 3), np.nan, np.float32)
    return kp, desc, xyz
