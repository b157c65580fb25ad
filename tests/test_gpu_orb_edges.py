"""The CUDA ORB (Kp/DetectorStrategy=2) at the edges of its parameters against cv::ORB through the oracle's RTAB-Map wrapper logic
(oracle/feature2d_py.py): feature counts down to levels with no quota and up to kMaxFrameQueries, runs of tied Harris responses, keypoints
against the borders of every pyramid level, the FAST threshold, real frames, the FAST candidate overflow and mixed batches.  Bar as in
test_gpu_orb.py: keypoints in order with responses and angles bit for bit, descriptor bytes and 3-D points.  Every case that reaches a
specialised kernel (TMA-staged FAST / blur, patch-staged descriptors, vectorised preparation) runs again with them switched off."""
from pathlib import Path

import cv2
import numpy as np
import pytest

from oracle import feature2d_py as f2d
from oracle import gftt_py as gf
from rtabmap_b200 import Engine, LcdError, synth
from rtabmap_b200.capi import DETECTOR_GFTT_ORB, DETECTOR_ORB

pytestmark = pytest.mark.gpu
K4 = synth.CAMERA_K4
GOLDEN = Path(__file__).parent / "golden"
LCD_ERR_INVALID, LCD_ERR_CAPACITY = -1, -3  # include/lcd_b200.h
SWITCHES = ("LCD_ORB_TMA", "LCD_ORB_PATCH", "LCD_ORB_PREP_VEC")


def check_frame(got, want):
    kp_g, d_g, x_g = got
    kp_w, d_w, x_w = want
    assert len(kp_g) == len(kp_w), (len(kp_g), len(kp_w))
    assert np.array_equal(kp_g.view(np.uint32), kp_w.view(np.uint32)), "keypoints differ"
    assert np.array_equal(d_g, d_w), f"{int(np.unpackbits(d_g ^ d_w).sum())} descriptor bits differ"
    assert np.array_equal(np.isnan(x_g), np.isnan(x_w))
    assert np.array_equal(np.nan_to_num(x_g).view(np.uint32), np.nan_to_num(x_w).view(np.uint32)), "3-D points differ"


def level_quotas(n_features, n_levels):
    """ORB computeKeyPoints' features per level (float arithmetic, cvRound)"""
    f = np.float32
    factor = f(0.5)
    nd = f(f(n_features) * (f(1) - factor) / (f(1) - f(0.5 ** n_levels)))
    q = []
    for _ in range(n_levels - 1):
        q.append(int(np.rint(nd)))
        nd = f(nd * factor)
    q.append(max(n_features - sum(q), 0))
    return q


def specialised_path(h, w, n_levels, edge, gftt=False):
    """lcd_orb_last_path of a detection with the specialised kernels allowed: 1 TMA tiles (every level's rows whole 16-byte vectors), 2
    patch-staged descriptors (edge >= kOrbPatchR = 19, every level's rows whole 4-byte words), 4 vectorised preparation, 8 GFTT/ORB"""
    levels = 1 if gftt else n_levels
    ws = [w >> l for l in range(levels)]
    stride = sum((w >> l) * (h >> l) for l in range(levels))
    path = 8 if gftt else 0
    if not gftt and all(x % 16 == 0 for x in ws):
        path |= 1
    if edge >= 19 and all(x % 4 == 0 for x in ws):
        path |= 2
    if w % 8 == 0 and h % 2 == 0 and stride % 16 == 0:
        path |= 4
    return path


def detect_both(monkeypatch, eng, imgs, depth, op, cap=0):
    """eng's detection of the batch, asserted equal, bit for bit, to the general kernels' (when the specialised ones ran)"""
    gftt = eng.detector()[0] == DETECTOR_GFTT_ORB
    h, w = imgs.shape[1:3]
    fast = eng.orb_detect_describe(imgs, depth, op, cap=cap)
    want = specialised_path(h, w, op.n_levels, op.edge_threshold, gftt)
    assert eng.orb_last_path == want
    if want & 7:
        with monkeypatch.context() as m:
            for name in SWITCHES:
                m.setenv(name, "0")
            general = eng.orb_detect_describe(imgs, depth, op, cap=cap)
            assert eng.orb_last_path == want & 8
        for a, b in zip(fast, general):
            check_frame(b, a)
    return fast


def sample_frames():
    z = np.load(GOLDEN / "samples_c1.npz")
    off = z["offsets"]
    return np.stack([cv2.imdecode(z["jpeg"][off[i]:off[i + 1]], cv2.IMREAD_COLOR) for i in range(len(off) - 1)])


def tie_grid(h, w, step, size, start):
    """identical squares: runs of exactly equal Harris responses"""
    g = np.zeros((h, w), np.uint8)
    for y in range(start, h - start, step):
        for x in range(start, w - start, step):
            g[y:y + size, x:x + size] = 200
    return g


def mosaic(h, w, block, seed):
    """random blocks, slightly blurred: over 4096 keypoints at every level count, under the 16384 FAST candidates a level holds"""
    rng = np.random.default_rng(seed)
    img = np.kron(rng.integers(0, 256, (h // block + 1, w // block + 1)).astype(np.uint8), np.ones((block, block), np.uint8))[:h, :w]
    return cv2.GaussianBlur(img, (3, 3), 0)


def border_frame(h, w, seed):
    """a synthetic scene with blocks of 1..8-pixel granularity laid against the four edges: corners near the border of every level"""
    rng = np.random.default_rng(seed)
    g = synth.make_image(h, w, seed).copy()
    for s in (1, 2, 4, 8):
        for _ in range(60):
            side = rng.integers(4)
            bw, bh = int(rng.integers(2, 6)) * s, int(rng.integers(2, 6)) * s
            d = int(rng.integers(0, 20)) * s
            if side == 0:
                y, x = d, int(rng.integers(0, w - bw))
            elif side == 1:
                y, x = h - bh - d, int(rng.integers(0, w - bw))
            elif side == 2:
                y, x = int(rng.integers(0, h - bh)), d
            else:
                y, x = int(rng.integers(0, h - bh)), w - bw - d
            y, x = max(0, min(y, h - bh)), max(0, min(x, w - bw))
            g[y:y + bh, x:x + bw] = rng.integers(0, 256)
    return g


def border_distance(kp, h, w):
    """(octave, distance in level pixels to the nearest edge of the keypoint's level) of every keypoint"""
    o = kp[:, 5].astype(int)
    x = (kp[:, 0] / 2.0 ** o).astype(int)
    y = (kp[:, 1] / 2.0 ** o).astype(int)
    return o, np.minimum.reduce([x, y, (w >> o) - 1 - x, (h >> o) - 1 - y])


# ---- feature counts x levels ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nf", [1, 2, 3, 7, 150, 1941, 1942, 2000, 3000, 4096])
@pytest.mark.parametrize("frame", ["synthetic", "real"])
def test_feature_counts_and_levels(monkeypatch, frame, nf):
    """Kp/MaxFeatures from levels whose quota rounds to 0 up to kMaxFrameQueries, where the merge of the levels' keypoints needs more
    than 48 KB of shared memory"""
    img = mosaic(720, 1280, 10, 8) if frame == "synthetic" else sample_frames()[33]
    eng = Engine()
    for lv in (1, 2, 3, 4):
        op = Engine.orb_params(K4, n_features=nf, n_levels=lv)
        got = detect_both(monkeypatch, eng, img[None], None, op, cap=min(nf + 256, 4096))[0]
        want = f2d.detect_describe(img, None, K4, f2d.OrbParams(n_features=nf, n_levels=lv))
        check_frame(got, want)
        for level, q in enumerate(level_quotas(nf, lv)):
            if q == 0:
                assert not (got[0][:, 5] == level).any(), (level, lv)
        if frame == "synthetic":
            assert len(want[0]) == nf  # more corners than the largest count: the merge cuts every frame
    if nf <= 3:
        assert 0 in level_quotas(nf, 4)


# ---- ties ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", [(9, 4, 24), (7, 3, 13)])
def test_tie_grid(monkeypatch, grid):
    """retainBest keeps every keypoint tied with a level's boundary response, here more than Kp/MaxFeatures of them; Feature2D::
    limitKeypoints then keeps the strongest, the later index first among equals"""
    g = tie_grid(480, 640, *grid)
    eng = Engine()
    for nf in (100, 300, 1000, 4096):
        p = f2d.OrbParams(n_features=nf)
        kps = f2d.make_orb(p).detect(g, None)
        per_level = np.bincount([k.octave for k in kps], minlength=3)
        assert len({k.response for k in kps}) <= 3 < len(kps) // 100, "the grid must tie"
        if nf <= 300:
            quota = level_quotas(nf, 3)
            assert any(per_level[l] > max(quota[l] + 256, nf) for l in range(3)), per_level
        got = detect_both(monkeypatch, eng, g[None], None, Engine.orb_params(K4, n_features=nf), cap=4096)[0]
        check_frame(got, f2d.detect_describe(g, None, K4, p))
    if grid == (7, 3, 13):
        assert per_level.max() > 4096  # a level keeps more than kMaxFrameQueries tied keypoints


# ---- borders -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("edge", [0, 3, 4, 5, 10, 14, 15, 16, 18, 19, 31, 64])
@pytest.mark.parametrize("detector", ["orb", "gftt"])
def test_edge_threshold(monkeypatch, detector, edge):
    """keypoints within 4 pixels of a level's edge take the Harris response on a reflected window, within 15 its IC angle on a reflected
    patch; below edge 19 the descriptors come from the general kernel; a level no larger than twice the edge comes back empty"""
    h, w = 480, 640
    img = border_frame(h, w, 3)
    depth = synth.make_depth(h, w, 4)
    p = f2d.OrbParams(n_features=1500, edge_threshold=edge)
    eng = Engine()
    if detector == "gftt":
        eng.set_detector(DETECTOR_GFTT_ORB)
        want = gf.detect_describe_gftt(img, depth, K4, p)
    else:
        want = f2d.detect_describe(img, depth, K4, p)
    got = detect_both(monkeypatch, eng, img[None], depth[None], Engine.orb_params(K4, n_features=1500, edge_threshold=edge))[0]
    check_frame(got, want)
    octave, dist = border_distance(want[0], h, w)
    for level in range(1 if detector == "gftt" else 3):
        at = octave == level
        if min(h, w) >> level <= 2 * edge:
            assert not at.any()
            continue
        assert at.any()
        if edge <= 3:
            assert (dist[at] < 4).any(), level
        if edge <= 14:
            assert (dist[at] < 15).any(), level


@pytest.mark.parametrize("edge", [19, 31])
@pytest.mark.parametrize("detector", ["orb", "gftt"])
def test_levels_at_most_twice_the_edge(monkeypatch, detector, edge):
    """120 x 160: level 2 (30 x 40) is no larger than twice either edge, level 1 (60 x 80) than twice 31"""
    img = border_frame(120, 160, 9)
    p = f2d.OrbParams(n_features=500, edge_threshold=edge)
    eng = Engine()
    if detector == "gftt":
        eng.set_detector(DETECTOR_GFTT_ORB)
        want = gf.detect_describe_gftt(img, None, K4, p)
    else:
        want = f2d.detect_describe(img, None, K4, p)
    got = detect_both(monkeypatch, eng, img[None], None, Engine.orb_params(K4, n_features=500, edge_threshold=edge))[0]
    check_frame(got, want)
    octaves = set(want[0][:, 5].astype(int).tolist())
    assert 0 in octaves
    if detector == "orb":
        assert 2 not in octaves and (1 not in octaves) == (edge == 31), octaves


# ---- FAST threshold ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("thr", [0, 1, 5, 40, 100, 254, 255])
def test_fast_threshold(monkeypatch, thr):
    """the general FAST kernel compares ints, the TMA kernel packs the threshold into four bytes: both at every 8-bit threshold"""
    eng = Engine()
    for img in (synth.make_image(720, 1280, 8), sample_frames()[0]):
        op = Engine.orb_params(K4, fast_threshold=thr)
        want = f2d.detect_describe(img, None, K4, f2d.OrbParams(fast_threshold=thr))
        check_frame(detect_both(monkeypatch, eng, img[None], None, op)[0], want)
        assert (len(want[0]) > 0) == (thr <= 100)


def small_dictionary_engine(detector=DETECTOR_ORB):
    vocab = synth.make_binary_vocabulary(2048, 32, 1)
    ids = np.arange(1, 2049, dtype=np.int32)
    smap = synth.make_map(ids, 50, 200, seed=2)
    eng = Engine(max_words=8192, max_signatures=400)
    eng.add_words(ids, vocab)
    eng.last_word_id = 2048
    eng.update()
    eng.load_csr(smap.word_ids, smap.row_ptr, smap.sig, smap.cnt)
    eng.set_detector(detector)
    return eng, smap


@pytest.mark.parametrize("thr", [-1, 256, 300])
def test_fast_threshold_out_of_range_is_rejected(thr):
    """cv::ORB takes FAST/Threshold modulo 256; the engine rejects what it cannot represent in 8 bits rather than emulate that"""
    img = synth.make_image(480, 640, 3)
    op = Engine.orb_params(K4, fast_threshold=thr)
    eng, smap = small_dictionary_engine()
    with pytest.raises(LcdError) as err:
        eng.orb_detect_describe(img[None], None, op)
    assert err.value.code == LCD_ERR_INVALID and "FAST/Threshold" in str(err.value), str(err.value)
    ns = len(smap.sig_ids)
    with pytest.raises(LcdError) as err:
        eng.process_frames(img[None], None, op, smap.sig_ids, ns + 1)
    assert err.value.code == LCD_ERR_INVALID and "FAST/Threshold" in str(err.value), str(err.value)
    check_frame(eng.orb_detect_describe(img[None], None, Engine.orb_params(K4))[0], f2d.detect_describe(img, None, K4, f2d.OrbParams()))


# ---- real frames ---------------------------------------------------------------------------------------------------------------------------
def test_sample_images(monkeypatch):
    """the 84 JPEG frames of samples_c1.npz in one batch"""
    imgs = sample_frames()
    eng = Engine()
    K = (400.0, 400.0, 256.0, 192.0)
    for nf in (1000, 150):
        out = detect_both(monkeypatch, eng, imgs, None, Engine.orb_params(K, n_features=nf))
        for i in range(len(imgs)):
            check_frame(out[i], f2d.detect_describe(imgs[i], None, K, f2d.OrbParams(n_features=nf)))


# ---- FAST candidate overflow ---------------------------------------------------------------------------------------------------------------
def check_fast_overflow(err):
    assert err.value.code == LCD_ERR_CAPACITY
    assert "16384 FAST corners" in str(err.value) and "FAST/Threshold" in str(err.value) and "GFTT" not in str(err.value), str(err.value)


def test_fast_candidate_overflow_is_reported():
    """uniform noise: ~30 000 level-0 FAST corners, more than the 16384 a level keeps.  Every image-level call fails with FAST's limit, and
    the flag clears on the next frame"""
    noise = np.random.default_rng(4).integers(0, 256, (480, 640), dtype=np.uint8)
    assert len(cv2.FastFeatureDetector_create(20, True).detect(noise)) > 16384
    img = synth.make_image(480, 640, 3)
    op = Engine.orb_params(K4)
    want = f2d.detect_describe(img, None, K4, f2d.OrbParams())
    eng = Engine()
    with pytest.raises(LcdError) as err:
        eng.orb_detect_describe(noise[None], None, op)
    check_fast_overflow(err)
    assert eng.orb_overflow()
    check_frame(eng.orb_detect_describe(img[None], None, op)[0], want)
    assert not eng.orb_overflow()

    # the calls that go on to the dictionary search, on a small dictionary and store
    eng, smap = small_dictionary_engine()
    ns = len(smap.sig_ids)
    with pytest.raises(LcdError) as err:
        eng.process_frames(noise[None], None, op, smap.sig_ids, ns + 1)
    check_fast_overflow(err)
    assert eng.orb_overflow()
    nkp = eng.process_frames(img[None], None, op, smap.sig_ids, ns + 1)[0]
    assert nkp[0] == len(want[0]) and not eng.orb_overflow()
    out = (np.zeros(1, np.int32), np.zeros((1, op.n_features), np.int32), np.zeros((1, ns), np.float32), np.zeros(1, np.int32), None)
    eng.process_frames_submit(noise[None], None, op, smap.sig_ids, ns + 1, None, *out)
    with pytest.raises(LcdError) as err:
        eng.process_frames_wait()
    check_fast_overflow(err)
    eng.map_detect_async(noise, None, op)
    with pytest.raises(LcdError) as err:
        eng.map_frame(ns + 1)
    check_fast_overflow(err)
    eng.map_detect_async(img, None, op)
    n_kp, _, _, _, _, desc, xyz = eng.map_frame(ns + 2, want_features=True)
    assert n_kp == len(want[0]) and not eng.orb_overflow()
    assert np.array_equal(desc, want[1]) and np.array_equal(xyz, want[2], equal_nan=True)


# ---- mixed batch ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nf", [300, 1000])
def test_mixed_batch(monkeypatch, nf):
    """a tie frame, a textureless frame, a border-heavy frame and a real frame in one call: each equals its detection alone and cv::ORB"""
    real = sample_frames()[17]
    h, w = real.shape[:2]
    gray = [tie_grid(h, w, 9, 4, 24), np.full((h, w), 7, np.uint8), border_frame(h, w, 5)]
    imgs = np.stack([cv2.cvtColor(g, cv2.COLOR_GRAY2BGR) for g in gray] + [real])
    depth = np.stack([synth.make_depth(h, w, 40 + i) for i in range(4)])
    op = Engine.orb_params(K4, n_features=nf)
    eng = Engine()
    batch = detect_both(monkeypatch, eng, imgs, depth, op)
    for i in range(4):
        want = f2d.detect_describe(imgs[i], depth[i], K4, f2d.OrbParams(n_features=nf))
        check_frame(batch[i], want)
        check_frame(eng.orb_detect_describe(imgs[i:i + 1], depth[i:i + 1], op)[0], want)
    assert len(batch[1][0]) == 0 and len(batch[0][0]) > 0
