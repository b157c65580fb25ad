"""Parity of the CUDA ORB (detect + describe + 3-D lifting) against OpenCV's cv::ORB — the third-party
implementation RTAB-Map's Feature2D calls (Features2d.cpp:1614/1657/1714) — through the oracle's restated
RTAB-Map wrapper logic (oracle/feature2d_py.py).  Bar: identical keypoints IN THE SAME ORDER (pt, octave,
size bit-exact; response and angle bit-exact floats), identical descriptor bytes, identical 3-D points."""
import numpy as np
import pytest

from oracle import feature2d_py as f2d
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import DETECTOR_GFTT_ORB

pytestmark = pytest.mark.gpu
K4 = synth.CAMERA_K4


def check_frame(got, want, exact_desc=True):
    kp_g, d_g, x_g = got
    kp_w, d_w, x_w = want
    assert len(kp_g) == len(kp_w), (len(kp_g), len(kp_w))
    assert np.array_equal(kp_g[:, [0, 1, 2, 5]], kp_w[:, [0, 1, 2, 5]]), "keypoint set / order differs"
    assert np.array_equal(kp_g[:, 4].view(np.uint32), kp_w[:, 4].view(np.uint32)), "Harris responses differ"
    assert np.array_equal(kp_g[:, 3].view(np.uint32), kp_w[:, 3].view(np.uint32)), "angles differ"
    bad_bits = int(np.unpackbits(d_g ^ d_w).sum())
    if exact_desc:
        assert bad_bits == 0, f"{bad_bits} descriptor bits differ"
    assert np.array_equal(np.isnan(x_g), np.isnan(x_w))
    assert np.array_equal(np.nan_to_num(x_g).view(np.uint32), np.nan_to_num(x_w).view(np.uint32)), "3-D points differ"
    return bad_bits


@pytest.mark.parametrize("seed", [5, 6, 7])
def test_orb_gray_with_depth_mask(seed):
    img = synth.make_image(480, 640, seed)
    depth = synth.make_depth(480, 640, seed + 10)
    eng = Engine()
    p = f2d.OrbParams()
    got = eng.orb_detect_describe(img[None], depth[None], Engine.orb_params(K4))[0]
    want = f2d.detect_describe(img, depth, K4, p)
    assert len(want[0]) > 900
    check_frame(got, want)


def test_orb_bgr_float_depth_batch():
    imgs = np.stack([synth.make_image(480, 640, 20 + i, bgr=True) for i in range(3)])
    depth = np.stack([synth.make_depth(480, 640, 30 + i, as_float=True) for i in range(3)])
    eng = Engine()
    got = eng.orb_detect_describe(imgs, depth, Engine.orb_params(K4, min_depth=0.5, max_depth=3.5))
    p = f2d.OrbParams(min_depth=0.5, max_depth=3.5)
    for i in range(3):
        check_frame(got[i], f2d.detect_describe(imgs[i], depth[i], K4, p))


def test_orb_no_depth_and_few_features():
    img = synth.make_image(240, 320, 3, n_rects=40)          # low texture: fewer corners than the quota
    eng = Engine()
    got = eng.orb_detect_describe(img[None], None, Engine.orb_params(K4, n_features=400, depth_as_mask=False))[0]
    want = f2d.detect_describe(img, None, K4, f2d.OrbParams(n_features=400, depth_as_mask=False))
    check_frame(got, want)
    assert np.isnan(got[2]).all()


def test_orb_limit_keypoints_when_levels_overflow_quota():
    # many equal Harris responses are unlikely; force the limit path with a smaller Kp/MaxFeatures than cv::ORB's own
    img = synth.make_image(480, 640, 11)
    eng = Engine()
    for nf, lv in ((500, 3), (300, 2), (1000, 1), (800, 4)):
        got = eng.orb_detect_describe(img[None], None, Engine.orb_params(K4, n_features=nf, n_levels=lv, depth_as_mask=False))[0]
        want = f2d.detect_describe(img, None, K4, f2d.OrbParams(n_features=nf, n_levels=lv, depth_as_mask=False))
        check_frame(got, want)


def test_orb_rejects_unsupported_parameters():
    from rtabmap_b200 import LcdError

    eng = Engine()
    img = np.zeros((1, 480, 640), np.uint8)
    with pytest.raises(LcdError):
        eng.orb_detect_describe(img, None, Engine.orb_params(K4, scale_factor=1.2))
    with pytest.raises(LcdError):
        eng.orb_detect_describe(np.zeros((1, 481, 641), np.uint8), None, Engine.orb_params(K4))


def test_process_frames_full_path_matches_oracle():
    """images -> detect -> quantise -> score -> verify through lcd_process_frames against cv2.ORB + the oracle."""
    from oracle import oracle_py as orc

    p = f2d.OrbParams(n_features=600)
    orb_fn = lambda img, dep: f2d.detect_describe(img, dep, K4, p)
    world = synth.make_place_world(orb_fn, n_places=5, n_words=2800, n_signatures=120, feats=600, height=240, width=320, seed=9)
    imgs, deps, places = synth.make_view_frames(world, 4, seed=5, max_shift=4)
    imgs[3] = 7            # a textureless frame: no keypoints at all
    eng = Engine()
    o = orc.OracleDictionary()
    for d in (eng, o):
        d.add_words(world.word_ids, world.vocab)
        d.last_word_id = int(world.word_ids.max())
        d.update()
        d.load_csr(world.smap.word_ids, world.smap.row_ptr, world.smap.sig, world.smap.cnt)
        d.set_ni(world.smap.sig_ids, world.smap.ni)
    eng.sig_add_batch(world.smap.sig_ids, world.store.desc, world.store.xyz, world.smap.ni)
    K4s = (262.5, 262.5, 160.0, 120.0)
    op = Engine.orb_params(K4s, n_features=600)
    vp = Engine.verify_params(K4s)
    nkp, words, like, hyp, res = eng.process_frames(imgs, deps, op, world.smap.sig_ids, 121, vp)
    p2 = f2d.OrbParams(n_features=600)
    for b in range(4):
        kp, d, x = f2d.detect_describe(imgs[b], deps[b], K4s, p2)
        assert nkp[b] == len(kp)
        if len(kp) == 0:
            assert not res[b]["ok"] and (words[b] == 0).all()
            continue
        w_o, l_o = o.localize_ro(d, world.smap.sig_ids, 121)
        assert np.array_equal(words[b][:len(w_o)], w_o) and (words[b][len(w_o):] == 0).all()
        assert np.allclose(like[b], l_o, atol=1e-4, rtol=1e-4)
        h = int(np.argmax(l_o))
        assert hyp[b] == world.smap.sig_ids[h] and world.sig_place[h] == places[b]
        n = int(world.smap.ni[h])
        v = orc.verify_pair(world.store.desc[h][:n], world.store.xyz[h][:n], d, kp[:, :2], K4s)
        assert res[b]["ok"] == v["ok"] and res[b]["n_matches"] == len(v["matches"]) and res[b]["n_inliers"] == len(v["inliers"])
        assert np.allclose(res[b]["rvec"], v["rvec"], atol=1e-4) and np.allclose(res[b]["tvec"], v["tvec"], atol=1e-4)
        assert res[b]["ok"]


def test_orb_1280x720():
    """BASELINE configs[2] frame size: same bar as 640x480 (keypoints, order, descriptors, 3-D points bit for bit)."""
    k4 = (910.0, 910.0, 640.0, 360.0)
    img = synth.make_image(720, 1280, 5)
    depth = synth.make_depth(720, 1280, 15)
    eng = Engine()
    got = eng.orb_detect_describe(img[None], depth[None], Engine.orb_params(k4))[0]
    want = f2d.detect_describe(img, depth, k4, f2d.OrbParams())
    assert len(want[0]) == 1000
    check_frame(got, want)


def check_general_kernels_equal_the_fast_paths(monkeypatch, eng, fast_path, general_path):
    imgs = np.stack([synth.make_image(480, 640, 40 + i, bgr=True) for i in range(2)])
    depth = np.stack([synth.make_depth(480, 640, 50 + i) for i in range(2)])
    op = Engine.orb_params(K4)
    fast = eng.orb_detect_describe(imgs, depth, op)
    assert eng.orb_last_path == fast_path
    for name in ("LCD_ORB_TMA", "LCD_ORB_PATCH", "LCD_ORB_PREP_VEC"):
        monkeypatch.setenv(name, "0")
    general = eng.orb_detect_describe(imgs, depth, op)
    assert eng.orb_last_path == general_path
    for a, b in zip(fast, general):
        for x, y in zip(a, b):
            assert np.array_equal(np.nan_to_num(x).view(np.uint8), np.nan_to_num(y).view(np.uint8))


def test_orb_general_kernels_equal_the_fast_paths(monkeypatch):
    """Every specialised kernel (TMA-staged FAST / blur, patch-staged descriptors, vectorised preparation) keeps its general predecessor
    as the fallback for shapes it does not cover; with the specialisations switched off the output must not change by a bit."""
    check_general_kernels_equal_the_fast_paths(monkeypatch, Engine(), 7, 0)


def test_gftt_general_kernels_equal_the_fast_paths(monkeypatch):
    """GFTT/ORB (path bit 8) shares the preparation and the descriptors with ORB, and so their switches: the same bar"""
    eng = Engine()
    eng.set_detector(DETECTOR_GFTT_ORB)
    check_general_kernels_equal_the_fast_paths(monkeypatch, eng, 14, 8)


@pytest.mark.parametrize("hw", [(252, 332), (244, 324)])
def test_orb_sizes_the_specialised_kernels_do_not_cover(hw):
    """(The engine needs sizes that are a multiple of 2^(levels-1).)  Rows that are not a multiple of 16 bytes (no tensor map), of 8 pixels (no vector loads) or, on a coarser level, of 4 bytes
    (no aligned patch loads): the general kernels run, same bar against cv::ORB."""
    h, w = hw
    img = synth.make_image(h, w, 61)
    depth = synth.make_depth(h, w, 62)
    eng = Engine()
    got = eng.orb_detect_describe(img[None], depth[None], Engine.orb_params(K4, n_features=400))[0]
    want = f2d.detect_describe(img, depth, K4, f2d.OrbParams(n_features=400))
    assert len(want[0]) > 100
    check_frame(got, want)
    assert eng.orb_last_path == 0
