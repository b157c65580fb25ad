"""The ORB-OCTREE restatement (oracle/orb_octree_py.py) on the CPU: the arithmetic of the CUDA resize and blur kernels against cv2, the
constructor's tables, the quadtree's rules (push to the front, the phase-2 cut, N = 0), the refusals, and the tie report on the sample
images (DESIGN.md §2)."""
from pathlib import Path

import cv2
import numpy as np
import pytest

from oracle import orb_octree_py as oc
from rtabmap_b200 import synth

GOLDEN = Path(__file__).parent / "golden"


def sample_grays():
    z = np.load(GOLDEN / "samples_c1.npz")
    off = z["offsets"]
    return [cv2.imdecode(z["jpeg"][off[i]:off[i + 1]], cv2.IMREAD_GRAYSCALE) for i in range(len(off) - 1)]


@pytest.mark.parametrize("factor", [2.0, 1.2, 1.5, 1.15, 3.0])
@pytest.mark.parametrize("h,w", [(480, 640), (720, 1280), (481, 643), (97, 131)])
def test_kernel_resize_equals_cv2(h, w, factor):
    img = synth.make_image(h, w, 5)
    src = img
    for _ in range(3):
        dw, dh = int(np.rint(np.float32(src.shape[1]) / np.float32(factor))), int(np.rint(np.float32(src.shape[0]) / np.float32(factor)))
        if dw < 2 or dh < 2:
            break
        want = cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(oc.kernel_resize(src, dw, dh), want)
        src = want


def test_kernel_blur_equals_cv2_on_contiguous_images():
    for img in sample_grays()[:12] + [synth.make_image(241, 333, 2), np.random.default_rng(3).integers(0, 256, (30, 31), dtype=np.uint8)]:
        want = cv2.GaussianBlur(img.copy(), (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101)
        assert np.array_equal(oc.kernel_blur(img), want)


def test_tables():
    scale, inv, per, umax = oc.tables(500, 2.0, 3)
    assert per == [286, 143, 71] and [float(s) for s in scale] == [1.0, 2.0, 4.0]
    assert umax == [15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3]
    _, _, per, _ = oc.tables(500, 1.2, 8)
    assert per == [109, 90, 75, 63, 52, 44, 36, 31] and sum(per) == 500
    for nf in (1, 3, 500, 1000, 4096):
        for f in (2.0, 1.2, 1.5, 1.15):
            for nl in range(1, 9):
                scale, inv, per, _ = oc.tables(nf, f, nl)
                assert len(per) == nl and min(per) >= 0 and sum(per) >= nf
                assert all(scale[i] == np.float32(scale[i - 1] * np.float32(f)) for i in range(1, nl))
    assert oc.tables(1, 1.2, 8)[2] == [0, 0, 0, 0, 0, 0, 0, 1]


def test_distribute_rules():
    # N = 0: one round of divisions, one key per node
    keys = [(x, y, float(10 + (x * 7 + y) % 5)) for y in range(4, 60, 9) for x in range(4, 90, 11)]
    sel0 = oc.distribute(keys, 100, 64, 0)
    assert 1 < len(sel0) <= 4 * 2
    # every node keeps its strongest key, the first in key order among equals; distinct keys
    sel = oc.distribute(keys, 100, 64, 20)
    assert len(set(sel)) == len(sel) and len(sel) >= 20
    # a single key: one node, never divided
    assert oc.distribute([(5, 5, 1.0)], 100, 64, 10) == [0]
    assert oc.distribute([], 100, 64, 10) == []
    # enough nodes for every key: all keys come back
    assert sorted(oc.distribute(keys, 100, 64, 10000)) == list(range(len(keys)))


def test_refusals():
    assert oc.check_params(640, 480, oc.OctreeParams()) is None
    assert oc.check_params(640, 480, oc.OctreeParams(scale_factor=1.2, n_levels=8)) is None
    assert oc.check_params(640, 480, oc.OctreeParams(n_levels=9)) == "ORB/NLevels"
    assert oc.check_params(640, 480, oc.OctreeParams(scale_factor=1.0)) == "ORB/ScaleFactor"
    assert oc.check_params(640, 480, oc.OctreeParams(scale_factor=float("nan"))) == "ORB/ScaleFactor"
    assert oc.check_params(640, 480, oc.OctreeParams(edge_threshold=18)) == "ORB/EdgeThreshold"
    assert oc.check_params(640, 480, oc.OctreeParams(patch_size=15)) == "ORB/PatchSize"
    assert oc.check_params(640, 480, oc.OctreeParams(n_levels=5)) == "level span"
    assert oc.check_params(200, 640, oc.OctreeParams(n_levels=1)) == "level aspect"
    assert oc.check_params(124, 124, oc.OctreeParams(n_levels=2)) is None
    assert oc.check_params(122, 122, oc.OctreeParams(n_levels=2)) == "level span"


needs_ref = pytest.mark.skipif(oc.ref_orbx_lib() is None, reason="oracle/_ref/libref_orbx.so is not built (no reference sources)")


@needs_ref
def test_tables_equal_the_compiled_reference():
    for nf in (1, 3, 500, 1000, 4096):
        for f in (2.0, 1.2, 1.5, 1.15):
            for nl in range(1, 9):
                scale, inv, per, umax = oc.tables(nf, f, nl)
                r_scale, r_inv, r_per, r_umax = oc.ref_tables(nf, f, nl)
                assert np.array_equal(np.array(scale, np.float32).view(np.uint32), np.array(r_scale, np.float32).view(np.uint32)), (nf, f, nl)
                assert np.array_equal(np.array(inv, np.float32).view(np.uint32), np.array(r_inv, np.float32).view(np.uint32)), (nf, f, nl)
                assert per == r_per and umax == r_umax, (nf, f, nl)


@needs_ref
def test_distribute_edges_equal_the_compiled_reference():
    rng = np.random.default_rng(4)
    keys = [(x, y, float(10 + (x * 7 + y) % 5)) for y in range(4, 60, 9) for x in range(4, 90, 11)]
    for n in (0, 1, 5, 20, 10000):  # N = 0: one round of divisions; a large N: every key comes back
        ev = []
        got = oc.distribute(keys, 100, 64, n, ev)
        if not ev:
            assert got == oc.ref_distribute(keys, 100, 64, n), n
    for w, h in ((100, 64), (64, 100), (250, 60), (37, 31)):  # one, two and four initial nodes
        pts = {(int(rng.integers(0, w)), int(rng.integers(0, h))) for _ in range(300)}
        ks = [(x, y, float(rng.integers(1, 4))) for x, y in sorted(pts, key=lambda p: (p[1], p[0]))]
        for n in (0, 3, 40, 150):
            ev = []
            got = oc.distribute(ks, w, h, n, ev)
            want = oc.ref_distribute(ks, w, h, n)
            if "set" not in ev:
                assert sorted(got) == sorted(want), (w, h, n)
            if not ev:
                assert got == want, (w, h, n)


@needs_ref
@pytest.mark.parametrize("cfg,expected", [(dict(), {"set": 61, "order": 50, None: 141}),
                                          (dict(scale_factor=1.2, n_levels=8), {"set": 468, "order": 111, None: 93})])
def test_distribute_equals_the_compiled_reference_on_sample_images(cfg, expected):
    """On the FAST keys of every level of the 84 C1 sample images, the restatement's DistributeOctTree equals the reference's own (set and
    order) on every level where no tie decided anything, and as a set where ties decided only the order; the tie counts are DESIGN §2's"""
    p = oc.OctreeParams(**cfg)
    _, inv, per, _ = oc.tables(p.n_features, p.scale_factor, p.n_levels)
    counts = {"set": 0, "order": 0, None: 0}
    for g in sample_grays():
        sizes = oc.level_sizes(g.shape[1], g.shape[0], inv)
        levels = [g]
        for lv in range(1, p.n_levels):
            levels.append(cv2.resize(levels[-1], sizes[lv], interpolation=cv2.INTER_LINEAR))
        for lv, img in enumerate(levels):
            keys = oc.fast_cells(img, p.edge_threshold, p.fast_threshold, p.fast_min_threshold)
            bw, bh = img.shape[1] - 2 * (p.edge_threshold - 3), img.shape[0] - 2 * (p.edge_threshold - 3)
            ev = []
            got = oc.distribute(keys, bw, bh, per[lv], ev)
            want = oc.ref_distribute(keys, bw, bh, per[lv])
            status = "set" if "set" in ev else ("order" if ev else None)
            counts[status] += 1
            if status is None:
                assert got == want
            elif status == "order":
                assert sorted(got) == sorted(want)
    assert counts == expected
