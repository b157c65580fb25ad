"""The GFTT/ORB detector (Kp/DetectorStrategy=8, lcd_detector_set) against cv::GFTTDetector + cv::ORB::compute through the oracle's
RTAB-Map wrapper logic (oracle/gftt_py.py): keypoints (all six fields, in order), descriptor bytes and 3-D points bit for bit, and the
switch reaching the image-level calls that compose detection with the descriptor-level ones."""
from pathlib import Path

import cv2
import numpy as np
import pytest

from oracle import feature2d_py as f2d
from oracle import gftt_py as gf
from rtabmap_b200 import Engine, LcdError, synth
from rtabmap_b200.capi import DEPTH_MASK_U8, DETECTOR_GFTT_ORB, DETECTOR_ORB

pytestmark = pytest.mark.gpu
K4 = synth.CAMERA_K4
GOLDEN = Path(__file__).parent / "golden"
LCD_ERR_CAPACITY = -3  # include/lcd_b200.h


def gftt_engine(**kw):
    eng = Engine()
    eng.set_detector(DETECTOR_GFTT_ORB, Engine.gftt_params(**kw))
    return eng


def check_frame(got, want):
    kp_g, d_g, x_g = got
    kp_w, d_w, x_w = want
    assert len(kp_g) == len(kp_w), (len(kp_g), len(kp_w))
    assert np.array_equal(kp_g.view(np.uint32), kp_w.view(np.uint32)), "keypoints differ"
    assert np.array_equal(d_g, d_w), f"{int(np.unpackbits(d_g ^ d_w).sum())} descriptor bits differ"
    assert np.array_equal(np.isnan(x_g), np.isnan(x_w))
    assert np.array_equal(np.nan_to_num(x_g).view(np.uint32), np.nan_to_num(x_w).view(np.uint32)), "3-D points differ"


def test_sample_images():
    z = np.load(GOLDEN / "samples_c1.npz")
    off = z["offsets"]
    imgs = np.stack([cv2.imdecode(z["jpeg"][off[i]:off[i + 1]], cv2.IMREAD_COLOR) for i in range(len(off) - 1)])
    eng = gftt_engine()
    K = (400.0, 400.0, 256.0, 192.0)
    for nf in (1000, 150):
        out = eng.orb_detect_describe(imgs, None, Engine.orb_params(K, n_features=nf))
        for i in range(len(imgs)):
            check_frame(out[i], gf.detect_describe_gftt(imgs[i], None, K, f2d.OrbParams(n_features=nf)))
    assert eng.orb_last_path & 8


@pytest.mark.parametrize("h,w,bgr,depth_kind", [(480, 640, False, "u16"), (480, 640, True, "f32"), (720, 1280, False, "u16"), (720, 1280, True, "mask"),
                                                 (240, 322, False, "none")])
def test_sizes_inputs_and_depth_types(h, w, bgr, depth_kind):
    img = synth.make_image(h, w, 5, bgr=bgr)
    depth = None
    kw = {}
    if depth_kind in ("u16", "f32"):
        depth = synth.make_depth(h, w, 15, as_float=depth_kind == "f32")
    elif depth_kind == "mask":
        depth = np.zeros((h, w), np.uint8)
        depth[:, : w // 2] = 255
        depth[h // 3:, w // 2:] = 1
        kw["depth_type"] = DEPTH_MASK_U8
    k4 = (500.0, 500.0, w / 2, h / 2)
    p = f2d.OrbParams(min_depth=0.3, max_depth=3.0) if depth_kind == "f32" else f2d.OrbParams()
    eng = gftt_engine()
    got = eng.orb_detect_describe(img[None], None if depth is None else depth[None],
                                  Engine.orb_params(k4, min_depth=p.min_depth, max_depth=p.max_depth), **kw)[0]
    want = gf.detect_describe_gftt(img, depth, k4, p)
    if depth_kind == "mask":  # a mask, not a depth image: the same keypoints, no 3-D points
        want = (want[0], want[1], np.full_like(want[2], np.nan))
    assert len(want[0]) > 300
    check_frame(got, want)


@pytest.mark.parametrize("nf", [1, 7, 500, 2000, 4096])
def test_feature_counts(nf):
    img = synth.make_image(720, 1280, 8)
    eng = gftt_engine()
    got = eng.orb_detect_describe(img[None], None, Engine.orb_params(K4, n_features=nf), cap=min(nf + 256, 4096))[0]
    check_frame(got, gf.detect_describe_gftt(img, None, K4, f2d.OrbParams(n_features=nf)))


def test_1920x1080_occupancy_bitmap_in_global_memory():
    img = synth.make_image(1080, 1920, 31, bgr=True)
    depth = synth.make_depth(1080, 1920, 32)
    k4 = (1400.0, 1400.0, 960.0, 540.0)
    eng = gftt_engine(quality_level=0.02)  # the default 0.001 leaves ~100 000 local maxima on this frame
    got = eng.orb_detect_describe(img[None], depth[None], Engine.orb_params(k4, n_features=2000))[0]
    check_frame(got, gf.detect_describe_gftt(img, depth, k4, f2d.OrbParams(n_features=2000), gf.GfttParams(quality_level=0.02)))


@pytest.mark.parametrize("q,md", [(0.01, 7.0), (0.001, 1.0), (0.001, 0.0), (0.001, 7.4), (0.05, 25.0)])
def test_gftt_parameters(q, md):
    img = synth.make_image(480, 640, 12)
    eng = gftt_engine(quality_level=q, min_distance=md)
    got = eng.orb_detect_describe(img[None], None, Engine.orb_params(K4, n_features=3000))[0]
    check_frame(got, gf.detect_describe_gftt(img, None, K4, f2d.OrbParams(n_features=3000), gf.GfttParams(q, md)))


def test_tie_grid():
    """identical squares: runs of exactly equal responses, ordered by the later raster position first"""
    g = np.zeros((480, 640), np.uint8)
    for y in range(24, 450, 9):
        for x in range(24, 610, 9):
            g[y:y + 4, x:x + 4] = 200
    eng = gftt_engine(min_distance=0.0)
    for nf in (100, 1000, 4096):
        want = gf.detect_describe_gftt(g, None, K4, f2d.OrbParams(n_features=nf), gf.GfttParams(min_distance=0.0))
        assert len(np.unique(want[0][:, 4])) < len(want[0]) // 4
        check_frame(eng.orb_detect_describe(g[None], None, Engine.orb_params(K4, n_features=nf), cap=4096)[0], want)


def test_batch_position_does_not_matter():
    imgs = np.stack([synth.make_image(480, 640, 60 + i, bgr=True) for i in range(4)])
    deps = np.stack([synth.make_depth(480, 640, 70 + i) for i in range(4)])
    eng = gftt_engine()
    op = Engine.orb_params(K4)
    a = eng.orb_detect_describe(imgs, deps, op)
    b = eng.orb_detect_describe(imgs[::-1].copy(), deps[::-1].copy(), op)
    for i in range(4):
        check_frame(a[i], b[3 - i])
        check_frame(a[i], gf.detect_describe_gftt(imgs[i], deps[i], K4, f2d.OrbParams()))


def check_gftt_overflow(err):
    assert err.value.code == LCD_ERR_CAPACITY
    assert "65536 GFTT candidates" in str(err.value) and "GFTT/QualityLevel" in str(err.value) and "FAST" not in str(err.value), str(err.value)


def test_candidate_overflow_is_reported():
    """a frame with more local maxima than the candidate list holds: every image-level call fails with GFTT's limit, and the flag clears
    on the next frame"""
    noise = np.random.default_rng(4).integers(0, 256, (1080, 1920), dtype=np.uint8)   # ~1 local maximum in 15 pixels: > 65 536
    eng = gftt_engine(min_distance=0.0)
    with pytest.raises(LcdError) as err:
        eng.orb_detect_describe(noise[None], None, Engine.orb_params(K4))
    check_gftt_overflow(err)
    assert eng.orb_overflow()
    img = synth.make_image(480, 640, 3)
    check_frame(eng.orb_detect_describe(img[None], None, Engine.orb_params(K4))[0],
                gf.detect_describe_gftt(img, None, K4, f2d.OrbParams(), gf.GfttParams(min_distance=0.0)))
    assert not eng.orb_overflow()

    # the calls that go on to the dictionary search, on a small dictionary and store
    vocab = synth.make_binary_vocabulary(2048, 32, 1)
    ids = np.arange(1, 2049, dtype=np.int32)
    smap = synth.make_map(ids, 50, 200, seed=2)
    eng = Engine(max_words=8192, max_signatures=400)
    eng.add_words(ids, vocab)
    eng.last_word_id = 2048
    eng.update()
    eng.load_csr(smap.word_ids, smap.row_ptr, smap.sig, smap.cnt)
    eng.set_detector(DETECTOR_GFTT_ORB, Engine.gftt_params(min_distance=0.0))
    op = Engine.orb_params(K4)
    ns = len(smap.sig_ids)
    with pytest.raises(LcdError) as err:
        eng.process_frames(noise[None], None, op, smap.sig_ids, ns + 1)
    check_gftt_overflow(err)
    out = (np.zeros(1, np.int32), np.zeros((1, op.n_features), np.int32), np.zeros((1, ns), np.float32), np.zeros(1, np.int32), None)
    eng.process_frames_submit(noise[None], None, op, smap.sig_ids, ns + 1, None, *out)
    with pytest.raises(LcdError) as err:
        eng.process_frames_wait()
    check_gftt_overflow(err)
    eng.map_detect_async(noise, None, op)
    with pytest.raises(LcdError) as err:
        eng.map_frame(ns + 1)
    check_gftt_overflow(err)


def test_switching_back_to_orb_and_parameters():
    img = synth.make_image(480, 640, 21)
    depth = synth.make_depth(480, 640, 22)
    op = Engine.orb_params(K4)
    eng = Engine()
    assert eng.detector()[0] == DETECTOR_ORB
    fast = eng.orb_detect_describe(img[None], depth[None], op)[0]
    eng.set_detector(DETECTOR_GFTT_ORB, Engine.gftt_params(min_distance=5.0))
    det, prm = eng.detector()
    assert det == DETECTOR_GFTT_ORB and prm.min_distance == 5.0
    check_frame(eng.orb_detect_describe(img[None], depth[None], op)[0],
                gf.detect_describe_gftt(img, depth, K4, f2d.OrbParams(), gf.GfttParams(min_distance=5.0)))
    for bad in (dict(use_harris=True), dict(block_size=5), dict(quality_level=-0.1), dict(quality_level=0.0), dict(min_distance=-1.0)):
        with pytest.raises(LcdError):
            eng.set_detector(DETECTOR_GFTT_ORB, Engine.gftt_params(**bad))
        assert eng.detector()[0] == DETECTOR_GFTT_ORB and eng.detector()[1].min_distance == 5.0
    with pytest.raises(LcdError):
        eng.set_detector(3)
    eng.set_detector(DETECTOR_ORB)
    check_frame(eng.orb_detect_describe(img[None], depth[None], op)[0], fast)
    check_frame(fast, f2d.detect_describe(img, depth, K4, f2d.OrbParams()))


def test_process_frames_detects_gftt():
    """lcd_process_frames with GFTT/ORB selected: its keypoint counts, words, likelihoods and registrations are those of
    lcd_orb_detect_describe composed with the oracle's quantisation, scoring and verification"""
    from oracle import oracle_py as orc

    K4s = (262.5, 262.5, 160.0, 120.0)
    p = f2d.OrbParams(n_features=600)
    orb_fn = lambda img, dep: gf.detect_describe_gftt(img, dep, K4, p)
    world = synth.make_place_world(orb_fn, n_places=5, n_words=2800, n_signatures=120, feats=600, height=240, width=320, seed=9)
    imgs, deps, places = synth.make_view_frames(world, 4, seed=5, max_shift=4)
    eng = gftt_engine()
    o = orc.OracleDictionary()
    for d in (eng, o):
        d.add_words(world.word_ids, world.vocab)
        d.last_word_id = int(world.word_ids.max())
        d.update()
        d.load_csr(world.smap.word_ids, world.smap.row_ptr, world.smap.sig, world.smap.cnt)
        d.set_ni(world.smap.sig_ids, world.smap.ni)
    eng.sig_add_batch(world.smap.sig_ids, world.store.desc, world.store.xyz, world.smap.ni)
    op = Engine.orb_params(K4s, n_features=600)
    vp = Engine.verify_params(K4s)
    nkp, words, like, hyp, res = eng.process_frames(imgs, deps, op, world.smap.sig_ids, 121, vp)
    det = gftt_engine().orb_detect_describe(imgs, deps, op)
    n_ok = 0
    for b in range(4):
        kp, d, x = gf.detect_describe_gftt(imgs[b], deps[b], K4s, p)
        check_frame(det[b], (kp, d, x))
        assert nkp[b] == len(kp)
        w_o, l_o = o.localize_ro(d, world.smap.sig_ids, 121)
        assert np.array_equal(words[b][:len(w_o)], w_o) and (words[b][len(w_o):] == 0).all()
        assert np.allclose(like[b], l_o, atol=1e-4, rtol=1e-4)
        h = int(np.argmax(l_o))
        assert hyp[b] == world.smap.sig_ids[h]
        n = int(world.smap.ni[h])
        v = orc.verify_pair(world.store.desc[h][:n], world.store.xyz[h][:n], d, kp[:, :2], K4s)
        assert res[b]["ok"] == v["ok"] and res[b]["n_matches"] == len(v["matches"]) and res[b]["n_inliers"] == len(v["inliers"])
        n_ok += int(res[b]["ok"])
    assert n_ok >= 2


def test_map_frame_detects_gftt():
    """lcd_map_detect_async + lcd_map_frame with GFTT/ORB selected equal lcd_orb_detect_describe + lcd_dict_quantize + lcd_index_score"""
    rng = np.random.default_rng(3)
    op = Engine.orb_params(K4, n_features=500)
    base = [(synth.make_image(240, 320, 900 + p, bgr=True), synth.make_depth(240, 320, 950 + p)) for p in range(3)]
    frames = [synth.render_view(*base[t % 3], int(rng.integers(-4, 5)), int(rng.integers(-4, 5)), 2.0, rng) for t in range(8)]
    pipe, seq = gftt_engine(), gftt_engine()
    for t in range(8):
        sig = t + 1
        pipe.map_detect_async(frames[t][0], frames[t][1], op)
        wm = np.arange(1, sig - 1, dtype=np.int32)
        n_kp, words, n_new, like, kp, desc, xyz = pipe.map_frame(sig, wm, sig, want_features=True)
        kp_s, desc_s, xyz_s = seq.orb_detect_describe(frames[t][0][None], frames[t][1][None], op, cap=500)[0]
        kp_o, d_o, x_o = gf.detect_describe_gftt(frames[t][0], frames[t][1], K4, f2d.OrbParams(n_features=500))
        assert n_kp == len(kp_o) and np.array_equal(desc, d_o) and np.array_equal(xyz, x_o, equal_nan=True)
        check_frame((kp_s, desc_s, xyz_s), (kp_o, d_o, x_o))
        seq.update()
        w_s, n_new_s = seq.quantize(desc_s, sig)
        assert np.array_equal(words, w_s) and n_new == n_new_s
        if len(wm):
            assert np.array_equal(like, seq.score(w_s, wm, sig))


def test_sharded_step_detects_gftt():
    """lcd_shard_process_frames_dev on a communicator of one rank with GFTT/ORB selected equals lcd_process_frames_dev on the same engine,
    and its words are those of the GFTT/ORB descriptors quantised by the descriptor-level call"""
    import torch

    K4s = (262.5, 262.5, 160.0, 120.0)
    p = f2d.OrbParams(n_features=600)
    world = synth.make_place_world(lambda img, dep: gf.detect_describe_gftt(img, dep, K4, p), n_places=5, n_words=2800, n_signatures=120,
                                   feats=600, height=240, width=320, seed=9)
    imgs, deps, _ = synth.make_view_frames(world, 4, seed=5, max_shift=4)
    eng = Engine(max_words=8192, max_signatures=400)
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = int(world.word_ids.max())
    eng.update()
    sm = world.smap
    eng.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    eng.set_ni(sm.sig_ids, sm.ni)
    eng.sig_add_batch(sm.sig_ids, world.store.desc, world.store.xyz, sm.ni)
    eng.set_detector(DETECTOR_GFTT_ORB, Engine.gftt_params())
    op = Engine.orb_params(K4s, n_features=600)
    vp = Engine.verify_params(K4s)
    nf, ns = len(imgs), len(sm.sig_ids)
    d_img = torch.from_numpy(imgs).cuda()
    d_dep = torch.from_numpy(deps.view(np.int16)).cuda()
    d_sig = torch.from_numpy(sm.sig_ids).cuda()
    d_rowids = torch.from_numpy(world.word_ids).cuda()
    ext = torch.cuda.ExternalStream(eng.stream)
    with torch.cuda.stream(ext):
        w0 = torch.zeros(nf * 600, dtype=torch.int32, device="cuda")
        l0 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        eng.process_frames_dev(d_img.data_ptr(), nf, 320, 240, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, ns + 1, vp, w0.data_ptr(),
                               l0.data_ptr(), True, 0.8, True)
        hyp0, res0 = eng.process_fetch(nf)
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        w1 = torch.zeros(nf * 600, dtype=torch.int32, device="cuda")
        l1 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        eng.shard_process_frames_dev(d_img.data_ptr(), nf, 320, 240, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, ns + 1, d_rowids.data_ptr(),
                                     int(world.word_ids.max()), vp, w1.data_ptr(), l1.data_ptr(), True, 0.8, True)
        hyp1, res1 = eng.process_fetch(nf)
        eng.shard_comm_destroy()
    assert torch.equal(w0, w1) and torch.equal(l0, l1) and np.array_equal(hyp0, hyp1)
    for a, c in zip(res0, res1):
        assert a["ok"] == c["ok"] and a["n_inliers"] == c["n_inliers"] and a["tvec"].tobytes() == c["tvec"].tobytes()
    from oracle import oracle_py as orc

    words = w0.view(nf, 600).cpu().numpy()
    o = orc.OracleDictionary()
    o.add_words(world.word_ids, world.vocab)
    o.last_word_id = int(world.word_ids.max())
    o.update()
    o.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    o.set_ni(sm.sig_ids, sm.ni)
    for b in range(nf):
        kp, d, _ = gf.detect_describe_gftt(imgs[b], deps[b], K4s, p)
        w_o, _ = o.localize_ro(d, sm.sig_ids, ns + 1)
        assert np.array_equal(words[b][:len(w_o)], w_o) and (words[b][len(w_o):] == 0).all(), b
    assert sum(r["ok"] for r in res0) >= 2
    eng.close()
