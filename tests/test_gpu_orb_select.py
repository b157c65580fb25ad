"""The ORB keypoint selection (orb_order_kernel, orb_harris_kernel, orb_rank_kernel, orb_angle_kernel) against cv::ORB through the oracle's
RTAB-Map wrapper logic, bit for bit per frame (keypoints in order with responses and angles, descriptors, 3-D points): the benchmark's 128
frames in one call, frames whose level-0 survivors of the first retainBest outnumber what a rank CTA holds in shared memory, levels without
a single FAST corner beside full frames, and a level-0 candidate list exactly at its capacity and one corner past it."""
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import feature2d_py as f2d
from rtabmap_b200 import Engine, LcdError, synth

pytestmark = pytest.mark.gpu
K4 = synth.CAMERA_K4
H, W = 480, 640
CAND_CAP = 16384     # kOrbCandCap: FAST corners a level-0 list holds
RANK_CAP = 4096      # kOrbRankCap: survivors a rank CTA holds in shared memory
LCD_ERR_CAPACITY = -3


def check_frame(got, want):
    kp_g, d_g, x_g = got
    kp_w, d_w, x_w = want
    assert len(kp_g) == len(kp_w), (len(kp_g), len(kp_w))
    assert np.array_equal(kp_g.view(np.uint32), kp_w.view(np.uint32)), "keypoints differ"
    assert np.array_equal(d_g, d_w), f"{int(np.unpackbits(d_g ^ d_w).sum())} descriptor bits differ"
    assert np.array_equal(np.isnan(x_g), np.isnan(x_w))
    assert np.array_equal(np.nan_to_num(x_g).view(np.uint32), np.nan_to_num(x_w).view(np.uint32)), "3-D points differ"


def counters(eng, n_frames, which):
    """per (frame, level) counters of the last detection: 4 FAST candidates, 6 survivors of retainBest(2N)"""
    return eng.debug_orb_buffer(which, n_frames * 3 * 4, np.int32).reshape(n_frames, 3)


def dot_frame(values, seed=0):
    """isolated one-pixel dots on black, 4 pixels apart inside the ORB border: every dot is exactly one level-0 FAST corner, of score
    value - 1, and dots of value <= 80 leave no corner on the coarser levels (a 2x2 average of at most 20)"""
    g = np.zeros((H, W), np.uint8)
    ys, xs = np.meshgrid(np.arange(20, H - 20, 4), np.arange(20, W - 20, 4), indexing="ij")
    assert len(values) <= ys.size
    order = np.random.default_rng(seed).permutation(ys.size)[:len(values)]
    g[ys.reshape(-1)[order], xs.reshape(-1)[order]] = values
    return g


def bench_frames(n):
    """the first batch of bench.py's query frames (its place images and depths, its pool seed)"""
    world = SimpleNamespace(images=np.stack([synth.make_image(H, W, 100 + p, bgr=True) for p in range(50)]),
                            depths=np.stack([synth.make_depth(H, W, 200 + p, zero_frac=0.01) for p in range(50)]))
    imgs, deps, _ = synth.make_view_frames(world, 3 * n, seed=3, mode="revisit")
    return imgs[:n], deps[:n]


def test_bench_batch():
    """128 frames in one call: two level-0 order CTAs per SM and the other levels' selection beside them"""
    imgs, deps = bench_frames(128)
    eng = Engine()
    op = Engine.orb_params(K4, n_features=1000)
    got = eng.orb_detect_describe(imgs, deps, op, cap=1000)
    assert not eng.orb_overflow()
    p = f2d.OrbParams(n_features=1000)
    for i in range(len(imgs)):
        check_frame(got[i], f2d.detect_describe(imgs[i], deps[i], K4, p))
    assert (counters(eng, 128, 6)[:, 0] >= 2 * 571).all()  # every frame's level 0 reaches its quota of 2N survivors


@pytest.mark.parametrize("nf", [300, 1000])
def test_survivors_past_rank_capacity(nf):
    """tied FAST scores at the retainBest(2N) boundary: every dot of the weakest kind survives, more than RANK_CAP of them, and the rank
    replay runs on its global workspace; the same frame beside a bench frame whose survivors stay in shared memory"""
    values = np.array([100] * 150 + [80] * 150 + [60] * 5700, np.uint8)  # 300 stronger dots: fewer than 2N at either count
    dots = dot_frame(values, 1)
    bench, _ = bench_frames(1)
    imgs = np.stack([np.repeat(dots[..., None], 3, 2), bench[0]])
    eng = Engine()
    got = eng.orb_detect_describe(imgs, None, Engine.orb_params(K4, n_features=nf))
    surv = counters(eng, 2, 6)
    assert counters(eng, 2, 4)[0, 0] == len(values)
    assert surv[0, 0] == len(values) > RANK_CAP, surv
    assert surv[1, 0] <= RANK_CAP, surv
    p = f2d.OrbParams(n_features=nf)
    for i in range(2):
        check_frame(got[i], f2d.detect_describe(imgs[i], None, K4, p))


def test_levels_without_candidates():
    """a flat frame (no corner on any level) and a dot frame (corners on level 0 only) between two full frames"""
    imgs, deps = bench_frames(2)
    gray = [np.full((H, W), 7, np.uint8), dot_frame(np.full(3000, 60, np.uint8), 2)]
    batch = np.stack([imgs[0]] + [np.repeat(g[..., None], 3, 2) for g in gray] + [imgs[1]])
    depth = np.stack([deps[0], deps[0], deps[0], deps[1]])
    depth[1:3] = 1000  # every pixel valid
    eng = Engine()
    op = Engine.orb_params(K4, n_features=1000)
    got = eng.orb_detect_describe(batch, depth, op)
    cand = counters(eng, 4, 4)
    assert (cand[[0, 3]] > 0).all() and (cand[1] == 0).all(), cand
    assert cand[2, 0] == 3000 and (cand[2, 1:] == 0).all(), cand
    p = f2d.OrbParams(n_features=1000)
    for i in range(4):
        check_frame(got[i], f2d.detect_describe(batch[i], depth[i], K4, p))
    assert len(got[1][0]) == 0 and len(got[2][0]) > 0


def test_candidate_cap():
    """CAND_CAP tied level-0 corners fill the list exactly and select as cv::ORB does (all of them survive retainBest(2N) and reach the rank
    replay); one corner more is reported as an overflow, and the flag clears on the next call"""
    eng = Engine()
    op = Engine.orb_params(K4, n_features=1000)
    full = dot_frame(np.full(CAND_CAP, 60, np.uint8), 3)
    got = eng.orb_detect_describe(full[None], None, op)[0]
    assert not eng.orb_overflow()
    assert counters(eng, 1, 4)[0, 0] == CAND_CAP and counters(eng, 1, 6)[0, 0] == CAND_CAP
    check_frame(got, f2d.detect_describe(full, None, K4, f2d.OrbParams(n_features=1000)))
    over = dot_frame(np.full(CAND_CAP + 1, 60, np.uint8), 3)
    with pytest.raises(LcdError) as err:
        eng.orb_detect_describe(over[None], None, op)
    assert err.value.code == LCD_ERR_CAPACITY and "16384 FAST corners" in str(err.value), str(err.value)
    assert eng.orb_overflow()
    check_frame(eng.orb_detect_describe(full[None], None, op)[0], got)
    assert not eng.orb_overflow()
