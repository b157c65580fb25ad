"""The GFTT/ORB detector (Kp/DetectorStrategy=8) at the edges of its kernels (rtabmap_b200/csrc/gftt.cuh), against cv::GFTTDetector +
cv::ORB::compute (oracle/gftt_py.detect_describe_gftt): keypoints (all six fields), descriptor bytes and 3-D points bit for bit.

  * widths whose last w % 32 columns OpenCV's row filter computes without fused multiply-add, and widths around the corner kernel's
    126-column tiles;
  * candidate counts around the sort's 8192-key shared-memory chunk, its power-of-two padding and the 65 536-candidate cap;
  * the 32-lane groups of the minDistance walk and the Kp/MaxFeatures cut inside and on the edges of a group;
  * the occupancy bitmap at the 200 KiB shared-memory limit and just above it;
  * masks, and a quality level that keeps only the maximum and its ties.

Every case asserts, on the CPU, that its frames reach the edge it is about, so that none passes vacuously."""
import cv2
import numpy as np
import pytest

from oracle import feature2d_py as f2d
from oracle import gftt_py as gf
from rtabmap_b200 import Engine, LcdError, synth
from rtabmap_b200.capi import DEPTH_MASK_U8, DETECTOR_GFTT_ORB
from test_gpu_gftt import check_frame, check_gftt_overflow

pytestmark = pytest.mark.gpu
K4 = synth.CAMERA_K4


def gftt_engine(**kw):
    eng = Engine()
    eng.set_detector(DETECTOR_GFTT_ORB, Engine.gftt_params(**kw))
    return eng


def tail_changed(g):
    """pixels whose lambda differs between OpenCV's map (unfused row pass in the last w % 32 columns) and one fused in every column"""
    return gf.corner_min_eig(g).view(np.uint32) != gf.corner_min_eig(g, simd_width=1).view(np.uint32)


def walk(g, mask, n, q, md):
    """the minDistance walk of goodFeaturesToTrack over the restatement's sorted candidates: (candidate x, y in walk order, kept flags,
    number walked, number of candidates suppressed by a kept candidate earlier in the same 32-candidate group)"""
    eig = gf.corner_min_eig(g)
    allc = gf.select_corners(eig, mask, 0, q, 0.0)  # every candidate, in sort order
    xs, ys = allc[:, 0].astype(int), allc[:, 1].astype(int)
    kept = np.zeros(len(allc), bool)
    in_group = 0
    walked = 0
    for i in range(len(allc)):
        if n > 0 and kept.sum() == n:
            break
        walked += 1
        if md < 1:
            kept[i] = True
            continue
        d2 = (xs[:i] - xs[i]) ** 2 + (ys[:i] - ys[i]) ** 2
        hit = kept[:i] & (d2 < md * md)
        kept[i] = not hit.any()
        in_group += int(hit[i - i % 32:].any())
    return xs, ys, kept, walked, in_group


def run_and_compare(eng, imgs, n_features=1000, edge=19, g=gf.GfttParams(), masks=None):
    op = Engine.orb_params(K4, n_features=n_features, edge_threshold=edge)
    p = f2d.OrbParams(n_features=n_features, edge_threshold=edge)
    cap = min(n_features + 256, 4096)
    if masks is None:
        got = eng.orb_detect_describe(imgs, None, op, cap=cap)
    else:
        got = eng.orb_detect_describe(imgs, masks, op, cap=cap, depth_type=DEPTH_MASK_U8)
    wants = []
    for i in range(len(imgs)):
        want = gf.detect_describe_gftt(imgs[i], None if masks is None else masks[i], K4, p, g)
        if masks is not None:  # a mask, not a depth image: no 3-D points
            want = (want[0], want[1], np.full_like(want[2], np.nan))
        check_frame(got[i], want)
        wants.append(want)
    return wants


# -- widths -------------------------------------------------------------------------------------------------------------------------

WIDTH_FEATURES = 4000  # enough corners that the strongest reach the few tail pixels whose lambda the unfused form changes
WIDTHS = [(240, 424), (360, 650), (480, 752), (480, 848), (600, 1000), (96, 124), (96, 126), (96, 128), (96, 252), (96, 254), (96, 380)]
SEEDS = (1, 3, 4, 5)


def border_filter(c, w, h, edge):
    return c[(c[:, 0] >= edge) & (c[:, 0] < w - edge) & (c[:, 1] >= edge) & (c[:, 1] < h - edge)]


def width_reached(imgs, edge):
    """w % 32 > edge: for some frame, the corners kept from a corner map fused in every column differ (after ORB's border filter) from
    cv2's, so a kernel without the unfused tail fails the case.  A tail no wider than the border (edge 19 at 424, 650, 752, 848, 1000)
    lies inside the border: these cases check that the border filter drops the tail's corners, and that the corners they suppress are
    those cv2 suppresses, but do not separate the two forms.  Widths that are multiples of 32 (128): a corner kept by the walk next to
    the boundary of the corner kernel's two tiles (columns 125 and 126)."""
    h, w = imgs.shape[1:3]
    for img in imgs:
        walked = gf.select_corners(gf.corner_min_eig(img), None, WIDTH_FEATURES, 0.001, 7.0)
        if w % 32 > edge:
            fused = border_filter(gf.select_corners(gf.corner_min_eig(img, simd_width=1), None, WIDTH_FEATURES, 0.001, 7.0), w, h, edge)
            kept = border_filter(walked, w, h, edge)
            if len(kept) != len(fused) or not np.array_equal(kept.view(np.uint32), fused.view(np.uint32)):
                return True
        elif w % 32:
            if tail_changed(img)[walked[:, 1].astype(int), walked[:, 0].astype(int)].any():
                return True
        elif np.isin(walked[:, 0], (125, 126)).any():
            return True
    return False


@pytest.mark.parametrize("edge", [3, 19])
@pytest.mark.parametrize("h,w", WIDTHS)
def test_widths(h, w, edge):
    """one batch of equal-size frames at a width that is not a multiple of 32 (or that splits into 126-column tiles)"""
    imgs = np.stack([synth.make_image(h, w, s) for s in SEEDS])
    run_and_compare(gftt_engine(), imgs, n_features=WIDTH_FEATURES, edge=edge)
    assert width_reached(imgs, edge), "no frame reaches the width's edge"


def test_process_frames_tail_width():
    """lcd_process_frames at 848x480 (16 tail columns, ORB/EdgeThreshold 3) with GFTT/ORB: its keypoint counts, words and likelihoods are
    those of cv2's detection composed with the oracle's quantisation and scoring"""
    from oracle import oracle_py as orc

    h, w = 480, 848
    K4s = (500.0, 500.0, w / 2, h / 2)
    p = f2d.OrbParams(n_features=600, edge_threshold=3)
    world = synth.make_place_world(lambda img, dep: gf.detect_describe_gftt(img, dep, K4s, p), n_places=5, n_words=2800, n_signatures=120,
                                   feats=600, height=h, width=w, seed=9)
    imgs, deps, _ = synth.make_view_frames(world, 4, seed=5, max_shift=4)
    eng = gftt_engine()
    o = orc.OracleDictionary()
    for d in (eng, o):
        d.add_words(world.word_ids, world.vocab)
        d.last_word_id = int(world.word_ids.max())
        d.update()
        d.load_csr(world.smap.word_ids, world.smap.row_ptr, world.smap.sig, world.smap.cnt)
        d.set_ni(world.smap.sig_ids, world.smap.ni)
    eng.sig_add_batch(world.smap.sig_ids, world.store.desc, world.store.xyz, world.smap.ni)
    op = Engine.orb_params(K4s, n_features=600, edge_threshold=3)
    nkp, words, like, _, _ = eng.process_frames(imgs, deps, op, world.smap.sig_ids, 121, Engine.verify_params(K4s))
    reached = False
    for b in range(len(imgs)):
        kp, d, x = gf.detect_describe_gftt(imgs[b], deps[b], K4s, p)
        gray = cv2.cvtColor(imgs[b], cv2.COLOR_BGR2GRAY)
        reached |= bool(tail_changed(gray)[kp[:, 1].astype(int), kp[:, 0].astype(int)].any())
        assert nkp[b] == len(kp)
        w_o, l_o = o.localize_ro(d, world.smap.sig_ids, 121)
        assert np.array_equal(words[b][:len(w_o)], w_o) and (words[b][len(w_o):] == 0).all()
        assert np.allclose(like[b], l_o, atol=1e-4, rtol=1e-4)
    assert reached, "no frame keeps a keypoint on a pixel the tail changes"


# -- candidate counts ---------------------------------------------------------------------------------------------------------------

DOT_H, DOT_W = 1080, 1920
# 215 x 383 sites, 3 to 5 pixels from the border: a dot reflected by the border would add a local maximum beside itself
SITES = np.stack(np.meshgrid(np.arange(3, DOT_H - 4, 5), np.arange(3, DOT_W - 4, 5), indexing="ij"), -1).reshape(-1, 2)
COUNTS = [0, 1, 2, 31, 32, 33, 4095, 4096, 8191, 8192, 8193, 16384, 16385, 32768, 32769, 65535, 65536]


def dot_frame(n, layout, seed=0):
    """n single-pixel dots on the pitch-5 lattice (one local maximum each) at brightness 60..255: "equal" (one tie run ordered by raster
    index), "increasing" with raster index (the strongest keys sort from the last candidates) or "shuffled" (seeded)."""
    rng = np.random.default_rng(seed + n)
    g = np.zeros((DOT_H, DOT_W), np.uint8)
    sel = SITES[np.sort(rng.choice(len(SITES), n, replace=False))]
    v = {"equal": np.full(n, 200), "increasing": 60 + (195 * np.arange(n)) // max(n - 1, 1)}.get(layout)
    if v is None:
        v = rng.permutation(60 + (195 * np.arange(n)) // max(n - 1, 1))
    g[sel[:, 0], sel[:, 1]] = v
    return g


def cv_candidates(g):
    c = cv2.goodFeaturesToTrack(g, 0, 0.001, 0)
    return 0 if c is None else len(c)


@pytest.fixture(scope="module")
def dot_engine():
    return gftt_engine(min_distance=0.0)


@pytest.mark.parametrize("layout", ["equal", "increasing", "shuffled"])
@pytest.mark.parametrize("n", COUNTS)
def test_candidate_counts(dot_engine, n, layout):
    g = dot_frame(n, layout)
    assert cv_candidates(g) == n
    want = run_and_compare(dot_engine, g[None], n_features=4096, g=gf.GfttParams(min_distance=0.0))[0]
    assert (len(want[0]) > 0) == (n > 0)


def test_candidate_cap_overflow(dot_engine):
    g = dot_frame(65537, "shuffled")
    assert cv_candidates(g) == 65537
    op = Engine.orb_params(K4, n_features=4096)
    with pytest.raises(LcdError) as err:
        dot_engine.orb_detect_describe(g[None], None, op, cap=4096)
    check_gftt_overflow(err)
    assert dot_engine.orb_overflow()
    run_and_compare(dot_engine, dot_frame(65536, "shuffled")[None], n_features=4096, g=gf.GfttParams(min_distance=0.0))
    assert not dot_engine.orb_overflow()


def test_mixed_batch(dot_engine):
    """a full candidate list, a flat frame, one dot and a real frame in one call: each frame equals its own detection and cv2"""
    real = np.zeros((DOT_H, DOT_W), np.uint8)
    real[300:780, 640:1280] = synth.make_image(480, 640, 11)
    frames = [dot_frame(65536, "shuffled", 1), np.full((DOT_H, DOT_W), 128, np.uint8), dot_frame(1, "equal", 2), real]
    assert [cv_candidates(f) for f in frames[:3]] == [65536, 0, 1] and 1000 < cv_candidates(real) < 65536
    imgs = np.stack(frames)
    g = gf.GfttParams(min_distance=0.0)
    wants = run_and_compare(dot_engine, imgs, n_features=4096, g=g)
    for i in range(len(imgs)):
        check_frame(dot_engine.orb_detect_describe(imgs[i:i + 1], None, Engine.orb_params(K4, n_features=4096), cap=4096)[0], wants[i])
    assert [len(w[0]) > 0 for w in wants] == [True, False, True, True]


# -- minDistance walk ---------------------------------------------------------------------------------------------------------------

def cluster_frame():
    """130 clusters of dots at pitch 2 and 3 on a 48-pixel grid, each cluster dimmer than the one before: the sort walks the clusters
    in turn, so the corners of one 32-candidate group lie close together and suppress each other"""
    rng = np.random.default_rng(17)
    g = np.zeros((480, 640), np.uint8)
    k = 0
    for cy in range(40, 440, 48):
        for cx in range(40, 600, 48):
            pitch = 2 + k % 2
            for y in range(cy - 8, cy + 9, pitch):
                for x in range(cx - 8, cx + 9, pitch):
                    g[y, x] = 254 - k + int(rng.integers(0, 2))
            k += 1
    return g


@pytest.mark.parametrize("nf", [31, 32, 33, 63, 64, 65])
@pytest.mark.parametrize("md", [0.5, 1.0, 1.5, 2.5, 7.0, 25.0, 1000.0])
def test_min_distance_walk(md, nf):
    g = cluster_frame()
    xs, ys, kept, walked, in_group = walk(g, None, nf, 0.001, md)
    if md > np.hypot(*g.shape):
        assert kept.sum() == 1 and len(xs) > 1
    else:
        assert kept.sum() == nf, "the Kp/MaxFeatures cut is not reached"
    if 2.5 <= md < 1000:
        assert in_group > 0, "no candidate is suppressed by a corner of its own 32-candidate group"
    want = run_and_compare(gftt_engine(min_distance=md), g[None], n_features=nf, g=gf.GfttParams(min_distance=md))[0]
    assert len(want[0]) > 0


# -- occupancy bitmap ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("md", [1.0, 7.0])
@pytest.mark.parametrize("h,w", [(1280, 1280), (1282, 1280), (2560, 640), (2562, 640)])
def test_occupancy_bitmap_limit(h, w, md):
    """ceil(w / 32) * h * 4 bytes: exactly 200 KiB keeps the bitmap in shared memory, two rows more move it to global memory"""
    assert ((w + 31) // 32 * h * 4 <= 200 * 1024) == (h in (1280, 2560))
    img = synth.make_image(h, w, h + w)
    q = 0.02  # the default 0.001 leaves more local maxima than the candidate list holds at these sizes
    assert cv_candidates_q(img, q) < 65536
    want = run_and_compare(gftt_engine(quality_level=q, min_distance=md), img[None], n_features=4096, g=gf.GfttParams(q, md))[0]
    assert (want[0][:, 1] >= h - 40).any(), "no kept corner in the bitmap's last rows"


def cv_candidates_q(g, q):
    c = cv2.goodFeaturesToTrack(g, 0, q, 0)
    return 0 if c is None else len(c)


# -- masks and quality ----------------------------------------------------------------------------------------------------------------

def test_mask_without_strongest_corner():
    """a dim frame with one bright square that the mask leaves out: the threshold comes from the strongest corner inside the mask"""
    img = (synth.make_image(480, 848, 21) // 4).astype(np.uint8)
    img[200:230, 400:430] = 255
    mask = np.full(img.shape, 255, np.uint8)
    mask[190:240, 390:440] = 0
    q = 0.05
    eig = gf.corner_min_eig(img)
    thr_all = np.float32(float(eig.max()) * q)
    assert eig[mask != 0].max() * 10 < eig.max()
    want = run_and_compare(gftt_engine(quality_level=q), img[None], g=gf.GfttParams(quality_level=q), masks=mask[None])[0]
    assert (want[0][:, 4] <= thr_all).sum() > 100, "too few kept corners below the threshold of the unmasked frame"


def test_mask_all_zero():
    img = synth.make_image(480, 848, 22)
    want = run_and_compare(gftt_engine(), img[None], masks=np.zeros((1,) + img.shape, np.uint8))[0]
    assert len(want[0]) == 0


def test_mask_tail_columns_only():
    img = synth.make_image(480, 848, 23)
    mask = np.zeros(img.shape, np.uint8)
    mask[:, 832:] = 255
    kp = run_and_compare(gftt_engine(), img[None], edge=3, masks=mask[None])[0][0]
    x, y = kp[:, 0].astype(int), kp[:, 1].astype(int)
    assert len(kp) and (x >= 832).all() and tail_changed(img)[y, x].any()


@pytest.mark.parametrize("md", [0.0, 7.0])
def test_quality_keeps_only_the_maximum_ties(md):
    """quality 0.999: identical squares tie at the maximum; a dimmer square and the rest fall below the threshold"""
    g = np.zeros((240, 320), np.uint8)
    for y in range(30, 200, 20):
        for x in range(30, 280, 20):
            g[y:y + 4, x:x + 4] = 200
    g[210:214, 150:154] = 150
    kp = run_and_compare(gftt_engine(quality_level=0.999, min_distance=md), g[None], n_features=4096, g=gf.GfttParams(0.999, md))[0][0]
    ref = gf.detect_describe_gftt(g, None, K4, f2d.OrbParams(n_features=4096), gf.GfttParams(0.001, md))[0]
    assert len(kp) > 1 and (kp[:, 4] == ref[:, 4].max()).all() and len(ref) > len(kp)
