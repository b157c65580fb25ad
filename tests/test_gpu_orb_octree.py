"""The ORB-OCTREE detector (Kp/DetectorStrategy=10, lcd_detector_set_orb_octree) against the restatement of RTAB-Map's ORBextractor
(oracle/orb_octree_py.py): keypoints (all six fields, in order), descriptor bytes and 3-D points bit for bit, the refusals, the device
cosf/sinf against the host libm, and the switch reaching the image-level calls that compose detection with the descriptor-level ones."""
import ctypes
from pathlib import Path

import cv2
import numpy as np
import pytest

from oracle import orb_octree_py as oc
from rtabmap_b200 import Engine, LcdError, synth
from rtabmap_b200.capi import DEPTH_MASK_U8, DETECTOR_ORB, DETECTOR_ORB_OCTREE, VerifyResult

pytestmark = pytest.mark.gpu
K4 = synth.CAMERA_K4
GOLDEN = Path(__file__).parent / "golden"
CONFIGS = {"2.0x3": dict(scale_factor=2.0, n_levels=3), "1.2x8": dict(scale_factor=1.2, n_levels=8), "1.5x5": dict(scale_factor=1.5, n_levels=5)}


def octree_engine(min_thr=7, **kw):
    eng = Engine(**kw)
    eng.set_detector_orb_octree(min_thr)
    return eng


def op_of(p: oc.OctreeParams, k4=K4):
    return Engine.orb_params(k4, n_features=p.n_features, n_levels=p.n_levels, scale_factor=p.scale_factor, edge_threshold=p.edge_threshold,
                             fast_threshold=p.fast_threshold, patch_size=p.patch_size, min_depth=p.min_depth, max_depth=p.max_depth,
                             depth_as_mask=p.depth_as_mask)


def check_frame(got, want):
    kp_g, d_g, x_g = got
    kp_w, d_w, x_w = want
    assert len(kp_g) == len(kp_w), (len(kp_g), len(kp_w))
    assert np.array_equal(kp_g.view(np.uint32), kp_w.view(np.uint32)), "keypoints differ"
    assert np.array_equal(d_g, d_w), f"{int(np.unpackbits(d_g ^ d_w).sum())} descriptor bits differ"
    assert np.array_equal(np.isnan(x_g), np.isnan(x_w))
    assert np.array_equal(np.nan_to_num(x_g).view(np.uint32), np.nan_to_num(x_w).view(np.uint32)), "3-D points differ"


def sample_images():
    z = np.load(GOLDEN / "samples_c1.npz")
    off = z["offsets"]
    return np.stack([cv2.imdecode(z["jpeg"][off[i]:off[i + 1]], cv2.IMREAD_COLOR) for i in range(len(off) - 1)])


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_sample_images(cfg):
    imgs = sample_images()
    p = oc.OctreeParams(**CONFIGS[cfg])
    eng = octree_engine()
    out = eng.orb_detect_describe(imgs, None, op_of(p), cap=1024)
    for i in range(len(imgs)):
        check_frame(out[i], oc.detect_describe_octree(imgs[i], None, K4, p))
    assert eng.orb_last_path == 16
    assert eng.detector()[0] == DETECTOR_ORB_OCTREE


@pytest.mark.parametrize("h,w,cfg", [(720, 1280, "2.0x3"), (720, 1280, "1.2x8"), (481, 643, "2.0x3"), (333, 517, "1.5x5"), (241, 321, "1.2x8")])
def test_sizes(h, w, cfg):
    img = synth.make_image(h, w, 11, bgr=True)
    p = oc.OctreeParams(n_features=1000, **CONFIGS[cfg])
    if oc.check_params(w, h, p):
        p = oc.OctreeParams(n_features=1000, scale_factor=CONFIGS[cfg]["scale_factor"], n_levels=2)
    got = octree_engine().orb_detect_describe(img[None], None, op_of(p), cap=2048)[0]
    check_frame(got, oc.detect_describe_octree(img, None, K4, p))


def test_smallest_levels():
    """the last level spans exactly 30 pixels inside ORB/EdgeThreshold - 3 in both directions; one pixel less is refused"""
    p = oc.OctreeParams(n_levels=2, scale_factor=2.0)
    # level 1 = 46 x 46: 46 - 2 * 16 = 14 < 30; level 1 of 124 x 124 = 62 - 32 = 30
    img = synth.make_image(124, 124, 3)
    assert oc.check_params(124, 124, p) is None and oc.check_params(122, 122, p) is not None
    eng = octree_engine()
    check_frame(eng.orb_detect_describe(img[None], None, op_of(p))[0], oc.detect_describe_octree(img, None, K4, p))
    with pytest.raises(LcdError):
        eng.orb_detect_describe(img[None, :122, :122].copy(), None, op_of(p))


def test_min_threshold_fallback_and_flat_image():
    img = synth.make_image(480, 640, 21)
    img[:, :320] = cv2.GaussianBlur(img[:, :320], (0, 0), 6) // 3 + 60  # low-contrast cells: FAST/Threshold finds nothing there
    for min_thr in (7, 1, 0):
        p = oc.OctreeParams(fast_min_threshold=min_thr)
        check_frame(octree_engine(min_thr).orb_detect_describe(img[None], None, op_of(p))[0], oc.detect_describe_octree(img, None, K4, p))
    flat = np.full((480, 640), 77, np.uint8)
    kp, d, x = octree_engine().orb_detect_describe(flat[None], None, op_of(oc.OctreeParams()))[0]
    assert len(kp) == 0


@pytest.mark.parametrize("kind", ["u16", "f32", "mask"])
def test_depth_masks(kind):
    h, w = 480, 640
    img = synth.make_image(h, w, 31, bgr=True)
    kw = {}
    if kind == "mask":
        depth = np.zeros((h, w), np.uint8)
        depth[:, : w // 2] = 255
        depth[h // 3:, w // 2:] = 1
        depth[::7, :] = 0  # rows that only the truncated coordinates of scaled levels fall on
        kw["depth_type"] = DEPTH_MASK_U8
    else:
        depth = synth.make_depth(h, w, 15, as_float=kind == "f32")
    p = oc.OctreeParams(n_features=800, scale_factor=1.2, n_levels=8, min_depth=0.3 if kind == "f32" else 0.0, max_depth=3.0 if kind == "f32" else 0.0)
    k4 = (500.0, 500.0, w / 2, h / 2)
    got = octree_engine().orb_detect_describe(img[None], depth[None], op_of(p, k4), **kw)[0]
    want = oc.detect_describe_octree(img, depth, k4, p, depth_is_mask=kind == "mask")
    full = oc.detect_describe_octree(img, None, k4, p)
    assert len(want[0]) < len(full[0]) and (want[0][:, 5] > 0).any()
    check_frame(got, want)


@pytest.mark.parametrize("nf", [1, 3, 100, 1000, 4096])
def test_max_features_cut(nf):
    """Kp/MaxFeatures cuts the output of all levels with FAST scores as responses: ties everywhere, the later index first"""
    img = synth.make_image(720, 1280, 8)
    p = oc.OctreeParams(n_features=nf, scale_factor=1.2, n_levels=8)
    got = octree_engine().orb_detect_describe(img[None], None, op_of(p), cap=min(nf + 256, 4096))[0]
    want = oc.detect_describe_octree(img, None, K4, p)
    assert len(want[0]) == nf
    check_frame(got, want)


def test_batches():
    imgs = sample_images()[:7]
    p = oc.OctreeParams(scale_factor=1.2, n_levels=8)
    want = [oc.detect_describe_octree(im, None, K4, p) for im in imgs]
    eng = octree_engine()
    for i in range(len(imgs)):
        check_frame(eng.orb_detect_describe(imgs[i:i + 1], None, op_of(p))[0], want[i])
    out = eng.orb_detect_describe(imgs, None, op_of(p))
    for i in range(len(imgs)):
        check_frame(out[i], want[i])
    big = np.concatenate([imgs] * 19)[:128]
    out = eng.orb_detect_describe(big, None, op_of(p))
    for i in range(128):
        check_frame(out[i], want[i % 7])


def test_refusals():
    img = synth.make_image(480, 640, 4)
    eng = octree_engine()
    for bad in (dict(n_levels=0), dict(n_levels=9), dict(scale_factor=1.0), dict(scale_factor=0.8), dict(scale_factor=float("inf")),
                dict(scale_factor=float("nan")), dict(edge_threshold=18), dict(patch_size=15), dict(fast_threshold=256),
                dict(scale_factor=2.0, n_levels=5)):  # level 4 = 40 x 30
        with pytest.raises(LcdError):
            eng.orb_detect_describe(img[None], None, Engine.orb_params(K4, **bad))
    tall = synth.make_image(640, 200, 4)  # span 168 x 608: round(0.28) = 0 initial nodes
    assert oc.check_params(200, 640, oc.OctreeParams(n_levels=1)) is not None
    with pytest.raises(LcdError):
        eng.orb_detect_describe(tall[None], None, Engine.orb_params(K4, n_levels=1))
    for bad in (-1, 256):
        with pytest.raises(LcdError):
            eng.set_detector_orb_octree(bad)
    assert eng.detector()[0] == DETECTOR_ORB_OCTREE
    with pytest.raises(LcdError):
        eng.set_detector(DETECTOR_ORB_OCTREE)
    eng.set_detector(DETECTOR_ORB)
    assert eng.detector()[0] == DETECTOR_ORB
    eng.set_detector_orb_octree(9)
    p = oc.OctreeParams(fast_min_threshold=9)
    check_frame(eng.orb_detect_describe(img[None], None, op_of(p))[0], oc.detect_describe_octree(img, None, K4, p))


_LIBM_FILL = r"""
#include <math.h>
#include <stdint.h>
#include <string.h>
void fill(uint32_t first, uint32_t count, float * c, float * s)
{
	for (uint32_t i = 0; i < count; ++i) { float x; uint32_t b = first + i; memcpy(&x, &b, 4); c[i] = cosf(x); s[i] = sinf(x); }
}
"""


def test_sincos_equals_host_libm(tmp_path):
    """the descriptor's cosf / sinf on the device equal the host libm's on every float in [0, 2 pi] (numpy's sin / cos are not libm's:
    the host values come from a C loop built here)"""
    import subprocess

    import torch

    src, so = tmp_path / "fill.c", tmp_path / "fill.so"
    src.write_text(_LIBM_FILL)
    subprocess.run(["cc", "-O2", "-fno-builtin", "-shared", "-fPIC", "-o", str(so), str(src), "-lm"], check=True)
    fill = ctypes.CDLL(str(so)).fill
    hi = int(np.array([6.2831855], np.float32).view(np.uint32)[0])
    eng = Engine()
    chunk = 1 << 25
    d_c = torch.empty(chunk, dtype=torch.float32, device="cuda")
    d_s = torch.empty(chunk, dtype=torch.float32, device="cuda")
    h_c = np.empty(chunk, np.float32)
    h_s = np.empty(chunk, np.float32)
    first = 0
    while first <= hi:
        n = min(chunk, hi + 1 - first)
        eng.debug_orb_sincos(first, n, d_c, d_s)
        fill(ctypes.c_uint32(first), ctypes.c_uint32(n), h_c.ctypes.data_as(ctypes.c_void_p), h_s.ctypes.data_as(ctypes.c_void_p))
        assert np.array_equal(d_c[:n].cpu().numpy().view(np.uint32), h_c[:n].view(np.uint32)), f"cosf differs from bit pattern {first:#x} on"
        assert np.array_equal(d_s[:n].cpu().numpy().view(np.uint32), h_s[:n].view(np.uint32)), f"sinf differs from bit pattern {first:#x} on"
        first += n


def _world(p):
    orb_fn = lambda img, dep: oc.detect_describe_octree(img, dep, K4, p)
    return synth.make_place_world(orb_fn, n_places=5, n_words=2800, n_signatures=120, feats=p.n_features, height=240, width=320, seed=9)


P_PIPE = oc.OctreeParams(n_features=600, n_levels=2, scale_factor=1.5)


def test_process_frames_detects_octree():
    """lcd_process_frames, and lcd_process_frames_submit + _wait, with ORB-OCTREE selected: counts, words, likelihoods and hypotheses of
    the restatement's features fed to the oracle's quantisation and scoring"""
    from oracle import oracle_py as orc

    K4s = (262.5, 262.5, 160.0, 120.0)
    p = P_PIPE
    world = _world(p)
    imgs, deps, places = synth.make_view_frames(world, 4, seed=5, max_shift=4)
    eng = octree_engine()
    o = orc.OracleDictionary()
    for d in (eng, o):
        d.add_words(world.word_ids, world.vocab)
        d.last_word_id = int(world.word_ids.max())
        d.update()
        d.load_csr(world.smap.word_ids, world.smap.row_ptr, world.smap.sig, world.smap.cnt)
        d.set_ni(world.smap.sig_ids, world.smap.ni)
    eng.sig_add_batch(world.smap.sig_ids, world.store.desc, world.store.xyz, world.smap.ni)
    op = op_of(p, K4s)
    vp = Engine.verify_params(K4s)
    nkp, words, like, hyp, res = eng.process_frames(imgs, deps, op, world.smap.sig_ids, 121, vp)
    # the pipelined pair lcd_process_frames_submit + _wait detects the same frames the same way
    out = (np.zeros(4, np.int32), np.zeros((4, p.n_features), np.int32), np.zeros((4, len(world.smap.sig_ids)), np.float32), np.zeros(4, np.int32),
           (VerifyResult * 4)())
    eng.process_frames_submit(imgs, deps, op, world.smap.sig_ids, 121, vp, *out)
    eng.process_frames_wait()
    assert np.array_equal(out[0], nkp) and np.array_equal(out[1], words) and np.array_equal(out[2], like) and np.array_equal(out[3], hyp)
    assert [r.ok for r in out[4]] == [r["ok"] for r in res] and [r.n_inliers for r in out[4]] == [r["n_inliers"] for r in res]
    for b in range(4):
        kp, d, x = oc.detect_describe_octree(imgs[b], deps[b], K4s, p)
        assert nkp[b] == len(kp)
        w_o, l_o = o.localize_ro(d, world.smap.sig_ids, 121)
        assert np.array_equal(words[b][:len(w_o)], w_o) and (words[b][len(w_o):] == 0).all()
        assert np.allclose(like[b], l_o, atol=1e-4, rtol=1e-4)
        assert hyp[b] == world.smap.sig_ids[int(np.argmax(l_o))]


def test_map_frame_detects_octree():
    """lcd_map_detect_async + lcd_map_frame with ORB-OCTREE selected equal lcd_orb_detect_describe + lcd_dict_quantize + lcd_index_score"""
    rng = np.random.default_rng(3)
    p = oc.OctreeParams(n_features=500, n_levels=2, scale_factor=1.2)
    op = op_of(p)
    base = [(synth.make_image(240, 320, 900 + i, bgr=True), synth.make_depth(240, 320, 950 + i)) for i in range(3)]
    frames = [synth.render_view(*base[t % 3], int(rng.integers(-4, 5)), int(rng.integers(-4, 5)), 2.0, rng) for t in range(8)]
    pipe, seq = octree_engine(), octree_engine()
    for t in range(8):
        sig = t + 1
        pipe.map_detect_async(frames[t][0], frames[t][1], op)
        wm = np.arange(1, sig - 1, dtype=np.int32)
        n_kp, words, n_new, like, kp, desc, xyz = pipe.map_frame(sig, wm, sig, want_features=True)
        kp_s, desc_s, xyz_s = seq.orb_detect_describe(frames[t][0][None], frames[t][1][None], op, cap=500)[0]
        kp_o, d_o, x_o = oc.detect_describe_octree(frames[t][0], frames[t][1], K4, p)
        assert n_kp == len(kp_o) and np.array_equal(desc, d_o) and np.array_equal(xyz, x_o, equal_nan=True)
        check_frame((kp_s, desc_s, xyz_s), (kp_o, d_o, x_o))
        seq.update()
        w_s, n_new_s = seq.quantize(desc_s, sig)
        assert np.array_equal(words, w_s) and n_new == n_new_s
        if len(wm):
            assert np.array_equal(like, seq.score(w_s, wm, sig))


def test_sharded_step_detects_octree():
    """lcd_shard_process_frames_dev on a communicator of one rank with ORB-OCTREE selected equals lcd_process_frames_dev"""
    import torch

    K4s = (262.5, 262.5, 160.0, 120.0)
    p = P_PIPE
    world = _world(p)
    imgs, deps, _ = synth.make_view_frames(world, 4, seed=5, max_shift=4)
    eng = Engine(max_words=8192, max_signatures=400)
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = int(world.word_ids.max())
    eng.update()
    sm = world.smap
    eng.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    eng.set_ni(sm.sig_ids, sm.ni)
    eng.sig_add_batch(sm.sig_ids, world.store.desc, world.store.xyz, sm.ni)
    eng.set_detector_orb_octree()
    op = op_of(p, K4s)
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
    from oracle import oracle_py as orc

    words = w0.view(nf, 600).cpu().numpy()
    o = orc.OracleDictionary()
    o.add_words(world.word_ids, world.vocab)
    o.last_word_id = int(world.word_ids.max())
    o.update()
    o.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    o.set_ni(sm.sig_ids, sm.ni)
    for b in range(nf):
        kp, d, _ = oc.detect_describe_octree(imgs[b], deps[b], K4s, p)
        w_o, _ = o.localize_ro(d, sm.sig_ids, ns + 1)
        assert np.array_equal(words[b][:len(w_o)], w_o) and (words[b][len(w_o):] == 0).all(), b
    eng.close()
