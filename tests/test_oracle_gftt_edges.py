"""The GFTT restatement (oracle/gftt_py.py) against the host's cv2 at the widths where OpenCV's vectorised row filter hands over to its
scalar tail: the vertical Sobel's row pass is fused only in the first (w // 32) * 32 columns.  The CUDA corner kernel follows the same
rule, so these tests pin the rule itself, and the probe fails loudly on a host whose OpenCV dispatches differently.  ORB's 7x7 blur goes
through the same float row filter, with the same rule (rtabmap_b200/csrc/orb.cuh, orb_blur_row)."""
import cv2
import numpy as np
import pytest

from oracle import gftt_py as gf
from oracle.gftt_py import _fma

S, S2 = np.float32(1.0 / 3060.0), np.float32(2.0 / 3060.0)
WIDE = [322, 424, 650, 752, 848, 1000, 1241]


def _noise(h, w, seed):
    return cv2.GaussianBlur(np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8), (5, 5), 1.5)


def _row_pass_forms(g):
    """dy with the row pass fused in every column, and unfused in every column"""
    P = np.pad(g, 1, mode="reflect").astype(np.float32)
    L, M, R = P[:, :-2], P[:, 1:-1], P[:, 2:]
    fused = _fma(R, S, _fma(M, S2, L * S))
    plain = (L * S + M * S2) + R * S
    return fused[2:] - fused[:-2], plain[2:] - plain[:-2]


@pytest.mark.parametrize("w", [40, 66, 100, 130, 424, 650, 752, 848, 1241])
def test_host_opencv_row_filter_tail_starts_at_multiple_of_32(w):
    g = np.random.default_rng(w).integers(0, 256, (256, w), dtype=np.uint8)
    cv_dy = cv2.Sobel(g, cv2.CV_32F, 0, 1, ksize=3, scale=1.0 / 3060.0)
    fused, plain = _row_pass_forms(g)
    x0 = (w // 32) * 32
    off = np.flatnonzero((cv_dy.view(np.uint32) != fused.view(np.uint32)).any(axis=0))
    assert (fused[:, x0] != plain[:, x0]).any(), "the probe image does not separate the two forms at the first tail column"
    assert len(off) and off[0] == x0, (
        f"this host's cv2 {cv2.__version__} leaves the fused row pass at column {off[0] if len(off) else None}, not {x0} = (w // 32) * 32: "
        "oracle/gftt_py.py and rtabmap_b200/csrc/gftt.cuh pin x86 opencv-python 4.13, whose AVX2 row filter is 32 pixels wide")
    assert np.array_equal(cv_dy[:, x0:].view(np.uint32), plain[:, x0:].view(np.uint32)), "the tail columns are not the unfused form"


def _check_map(g):
    eig = gf.corner_min_eig(g)
    ref = cv2.cornerMinEigenVal(g, 3, 3)
    bad = eig.view(np.uint32) != ref.view(np.uint32)
    assert not bad.any(), f"{int(bad.sum())} pixels differ, columns {sorted(set(np.nonzero(bad)[1].tolist()))[:8]}"
    return eig


@pytest.mark.parametrize("w", list(range(8, 131)) + WIDE)
def test_corner_map_every_width(w):
    g = np.random.default_rng(w).integers(0, 256, (48, w), dtype=np.uint8)
    eig = _check_map(g)
    if w > 32 and w % 32 >= 8:  # the tail matters on this image: the fused-everywhere map is not cv2's
        assert (eig.view(np.uint32) != gf.corner_min_eig(g, simd_width=1).view(np.uint32)).any()


@pytest.mark.parametrize("h,w", [(4096, 64), (64, 4096)])
def test_corner_map_long_sizes(h, w):
    """the running double column sum over 4096 rows, and 4096 columns of row pass with a 32-aligned width"""
    _check_map(_noise(h, w, h + 3 * w))


def _cv_corners(g, n, q, md):
    kps = cv2.GFTTDetector_create(n, q, md, 3, False, 0.04).detect(g, None)
    return np.array([[k.pt[0], k.pt[1], k.response] for k in kps], np.float32).reshape(-1, 3)


@pytest.mark.parametrize("md", [0.0, 1.0, 2.5, 7.0])
def test_selection_tail_heavy_width(md):
    """848x480 (RealSense): 16 tail columns; the kept corners and their responses equal cv2.GFTTDetector's, and some of them sit on
    pixels whose lambda the unfused tail changes"""
    from rtabmap_b200 import synth

    g = synth.make_image(480, 848, 3)
    eig = _check_map(g)
    fused = gf.corner_min_eig(g, simd_width=1)
    got = gf.select_corners(eig, None, 4096, 0.001, md)
    want = _cv_corners(g, 4096, 0.001, md)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    x, y = got[:, 0].astype(int), got[:, 1].astype(int)
    assert ((x >= 832) & (eig[y, x] != fused[y, x])).any(), "no kept corner on a pixel the tail changes"
    pts = cv2.goodFeaturesToTrack(g, 4096, 0.001, md).reshape(-1, 2)
    assert np.array_equal(got[:, :2], pts)


def _orb_blur(g, simd_width=32):
    """ORB's GaussianBlur(7x7, sigma 2, reflect-101) on a sub-matrix, i.e. the float sepFilter2D the kernels restate: row pass in plain
    order, fused in the first (w // simd_width) * simd_width columns and unfused in the rest; symmetric fused column pass; rounded to
    uint8 half to even"""
    k = cv2.getGaussianKernel(7, 2, cv2.CV_32F).ravel().astype(np.float32)
    h, w = g.shape
    P = np.pad(g, 3, mode="reflect").astype(np.float32)
    x0 = (w // simd_width) * simd_width
    fused = P[:, :w] * k[0]
    plain = fused.copy()
    for j in range(1, 7):
        fused = _fma(P[:, j:j + w], k[j], fused)
        plain = plain + P[:, j:j + w] * k[j]
    r = np.concatenate([fused[:, :x0], plain[:, x0:]], axis=1)
    c = r[3:3 + h] * k[3]
    for j in range(1, 4):
        c = _fma(r[3 + j:3 + j + h] + r[3 - j:3 - j + h], k[3 + j], c)
    return np.clip(np.rint(c), 0, 255).astype(np.uint8)


def test_orb_blur_row_filter_tail():
    """the blur restated with the unfused tail equals cv2's float separable filter bit for bit at tail-heavy widths; fused in every
    column it does not (96x250 and 96x252: one pixel each, in the tail, inside a kept corner's descriptor patch)"""
    from rtabmap_b200 import synth

    k = cv2.getGaussianKernel(7, 2, cv2.CV_32F).ravel().astype(np.float32)
    fused_off = 0
    for h, w, seeds in [(96, 250, (3,)), (96, 252, (3, 4, 5)), (96, 254, (3,)), (96, 380, (1,)), (480, 752, (3,)), (480, 848, (3,)),
                        (600, 1000, (3,))]:
        for seed in seeds:
            g = synth.make_image(h, w, seed)
            ref = cv2.sepFilter2D(g, cv2.CV_8U, k, k, borderType=cv2.BORDER_REFLECT_101)
            got = _orb_blur(g)
            assert np.array_equal(got, ref), f"{h}x{w} seed {seed}: {int((got != ref).sum())} pixels differ"
            fused_off += int((_orb_blur(g, simd_width=1) != ref).sum())
    for w in range(8, 131):
        g = np.random.default_rng(w).integers(0, 256, (40, w), dtype=np.uint8)
        assert np.array_equal(_orb_blur(g), cv2.sepFilter2D(g, cv2.CV_8U, k, k, borderType=cv2.BORDER_REFLECT_101)), w
    assert fused_off > 0, "no image separates the fused row pass from cv2's"
