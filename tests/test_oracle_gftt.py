"""The numpy restatement of GFTT (oracle/gftt_py.py) against OpenCV's own cornerMinEigenVal and GFTTDetector, bit for bit: the CUDA
kernels of the GFTT/ORB detector are written against this restatement."""
from pathlib import Path

import cv2
import numpy as np
import pytest

from oracle import gftt_py as gf

GOLDEN = Path(__file__).parent / "golden"


def _samples():
    z = np.load(GOLDEN / "samples_c1.npz")
    off = z["offsets"]
    return [cv2.cvtColor(cv2.imdecode(z["jpeg"][off[i]:off[i + 1]], cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY) for i in range(len(off) - 1)]


def _cv_corners(gray, mask, n, q, md):
    kps = cv2.GFTTDetector_create(n, q, md, 3, False, 0.04).detect(gray, mask)
    for k in kps:
        assert k.size == 3 and k.angle == -1 and k.octave == 0
    return np.array([[k.pt[0], k.pt[1], k.response] for k in kps], np.float32).reshape(-1, 3)


def _check(gray, mask=None, n=1000, q=0.001, md=7.0):
    eig = gf.corner_min_eig(gray)
    ref = cv2.cornerMinEigenVal(gray, 3, 3)
    assert np.array_equal(eig.view(np.uint32), ref.view(np.uint32)), f"{int((eig.view(np.uint32) != ref.view(np.uint32)).sum())} pixels differ"
    got = gf.select_corners(eig, mask, n, q, md)
    want = _cv_corners(gray, mask, n, q, md)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    return len(got)


def test_every_sample_image():
    for i, g in enumerate(_samples()):
        assert _check(g) > 0, i


def test_sample_images_cuts_and_distances():
    imgs = _samples()
    for g in imgs[::7]:
        for n, q, md in ((1, 0.001, 7.0), (150, 0.01, 7.0), (4096, 1e-6, 0.5), (500, 0.001, 1.0), (700, 0.001, 7.4), (300, 0.05, 20.0)):
            _check(g, None, n, q, md)


@pytest.mark.parametrize("h,w", [(480, 640), (720, 1280), (61, 97)])
def test_sizes(h, w):
    from rtabmap_b200 import synth

    g = synth.make_image(h, w, 3) if h >= 240 else cv2.GaussianBlur(np.random.default_rng(2).integers(0, 256, (h, w), dtype=np.uint8), (5, 5), 1.2)
    _check(g, n=4096, md=3.0)
    _check(g, n=4096, md=0.0)


def test_tie_grid():
    """identical squares: equal responses everywhere, the later raster position first"""
    g = np.zeros((240, 320), np.uint8)
    for y in range(20, 220, 9):
        for x in range(20, 300, 9):
            g[y:y + 4, x:x + 4] = 200
    assert _check(g, n=4096, md=0.0) > 100
    _check(g, n=500, md=5.0)
    _check(g, n=37, md=1.0)
    want = _cv_corners(g, None, 4096, 0.001, 0.0)
    assert len(np.unique(want[:, 2])) < len(want) // 10, "the grid should produce exact ties"


def test_masks():
    from rtabmap_b200 import synth

    g = synth.make_image(480, 640, 9)
    depth = synth.make_depth(480, 640, 19)
    from oracle import feature2d_py as f2d

    mask = f2d.depth_mask(depth, f2d.OrbParams())
    _check(g, mask)
    half = np.zeros_like(mask)
    half[:, 320:] = 255
    _check(g, half, n=300, md=10.0)
    _check(g, np.zeros_like(mask))
