"""Memory::createSignature's split on the GPU (lcd_quantize_limit_set): the Kp/MaxFeatures strongest keypoints of a frame are quantised,
every detected keypoint registers.  Each image-level call is compared with the oracle's composition (detect -> limit_keypoints_inliers ->
quantise the picked rows -> negative ids for the others), and the device primitives with the oracle directly."""
import ctypes

import numpy as np
import pytest

from oracle import limit_py as lk
from oracle import oracle_py as orc
from rtabmap_b200 import Engine, LcdError, synth
from rtabmap_b200.capi import DETECTOR_GFTT_ORB, DETECTOR_ORB, LCD_DESC_F32

pytestmark = pytest.mark.gpu

K4 = synth.CAMERA_K4
DET, K = 1000, 500          # Vis/MaxFeatures detected, Kp/MaxFeatures quantised
KP_DTYPE = np.dtype([("x", "f4"), ("y", "f4"), ("size", "f4"), ("angle", "f4"), ("response", "f4"), ("octave", "i4")])


def engine(detector=DETECTOR_ORB, **gftt):
    eng = Engine(max_words=16384, max_signatures=400)
    if detector == DETECTOR_GFTT_ORB:
        eng.set_detector(DETECTOR_GFTT_ORB, Engine.gftt_params(**gftt))
    return eng


def make_world(detector=DETECTOR_ORB):
    det = engine(detector)
    op = Engine.orb_params(K4, n_features=DET)
    return synth.make_place_world(lambda im, dp: det.orb_detect_describe(im[None], dp[None], op, cap=DET)[0], 4, 4000, 40, DET, 480, 640, seed=11)


@pytest.fixture(scope="module")
def world():
    return make_world()


def load(eng, world):
    sm = world.smap
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = int(world.word_ids.max())
    eng.update()
    eng.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    eng.set_ni(sm.sig_ids, sm.ni)
    eng.sig_add_batch(sm.sig_ids, world.store.desc, world.store.xyz, sm.ni)
    return eng


def oracle_dict(world):
    o = orc.OracleDictionary()
    sm = world.smap
    o.add_words(world.word_ids, world.vocab)
    o.last_word_id = int(world.word_ids.max())
    o.update()
    o.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    o.set_ni(sm.sig_ids, sm.ni)
    return o


def expected(o, kp, desc, sig_ids, n_total, max_features, ratio, mean):
    """the oracle's createSignature split: (word ids [n], likelihood [ns])"""
    like = np.zeros(len(sig_ids), np.float32)

    def quantize(raw):
        w, l_o = o.localize_ro(desc[raw], sig_ids, n_total)
        like[:] = l_o
        return w

    words, _ = lk.signature_word_ids(kp, max_features, ratio, mean, quantize)
    return words, like


def top(like, sig_ids):
    h = int(np.argmax(like))
    return (int(sig_ids[h]), h) if like[h] > 0 else (0, -1)


def grid_image(step=9, h=480, w=640):
    g = np.zeros((h, w), np.uint8)
    for y in range(24, h - 30, step):
        for x in range(24, w - 30, step):
            g[y:y + 4, x:x + 4] = 200
    return g


@pytest.mark.parametrize("detector", [DETECTOR_ORB, DETECTOR_GFTT_ORB])
def test_fused_call_quantises_the_strongest_and_registers_with_all(world, detector):
    if detector != DETECTOR_ORB:
        world = make_world(detector)   # stored signatures of the detector's own keypoints, so that frames register
    sm = world.smap
    n_total = len(sm.sig_ids) + 1
    eng = load(engine(detector), world)
    eng.set_quantize_limit(K, 0.5, K)
    assert eng.quantize_limit == (K, 0.5, K)
    imgs, deps, _ = synth.make_view_frames(world, 4, seed=5, max_shift=4)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    nkp, words, like, hyp, res = eng.process_frames(imgs, deps, op, sm.sig_ids, n_total, vp)
    det = engine(detector).orb_detect_describe(imgs, deps, op, cap=DET)
    o = oracle_dict(world)
    assert max(len(d[0]) for d in det) > K
    n_ok = 0
    for b in range(4):
        kp, d, _ = det[b]
        n = len(kp)
        assert nkp[b] == n
        w_o, l_o = expected(o, kp, d, sm.sig_ids, n_total, K, 0.5, K)
        assert np.array_equal(words[b][:n], w_o) and (words[b][n:] == 0).all()
        assert (words[b][:n] > 0).sum() == min(n, K)
        assert np.allclose(like[b], l_o, atol=1e-4, rtol=1e-4)
        hid, h = top(l_o, sm.sig_ids)
        assert hyp[b] == hid
        if h >= 0:
            ni = int(sm.ni[h])
            v = orc.verify_pair(world.store.desc[h][:ni], world.store.xyz[h][:ni], d, kp[:, :2], K4)
            assert res[b]["ok"] == v["ok"] and res[b]["n_matches"] == len(v["matches"]) and res[b]["n_inliers"] == len(v["inliers"])
            n_ok += int(res[b]["ok"])
    assert n_ok >= 2


def test_gftt_tie_run_cut_by_the_limit(world):
    """GFTT's tie grid: runs of equal responses, and K falls inside one (the later index is kept first)"""
    sm = world.smap
    n_total = len(sm.sig_ids) + 1
    g = grid_image()
    eng = load(engine(DETECTOR_GFTT_ORB, min_distance=0.0), world)
    eng.set_quantize_limit(K, 0.0, 0)
    op = Engine.orb_params(K4, n_features=DET)
    nkp, words, like, _, _ = eng.process_frames(g[None], None, op, sm.sig_ids, n_total)
    kp, d, _ = engine(DETECTOR_GFTT_ORB, min_distance=0.0).orb_detect_describe(g[None], None, op, cap=DET)[0]
    r = np.sort(np.abs(kp[:, 4]))[::-1]
    assert len(kp) == DET and r[K - 1] == r[K]
    w_o, l_o = expected(oracle_dict(world), kp, d, sm.sig_ids, n_total, K, 0.0, 0)
    assert nkp[0] == DET and np.array_equal(words[0], w_o)
    assert np.allclose(like[0], l_o, atol=1e-4, rtol=1e-4)


def test_limit_off_or_never_reached_changes_nothing(world):
    sm = world.smap
    n_total = len(sm.sig_ids) + 1
    eng = load(engine(), world)
    imgs, deps, _ = synth.make_view_frames(world, 3, seed=8, max_shift=4)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    base = eng.process_frames(imgs, deps, op, sm.sig_ids, n_total, vp)
    assert eng.quantize_limit == (0, 0.0, 0)
    for lim in ((0, 0.0, 0), (DET, 0.5, 2), (0, 0.5, 2)):   # off; every frame <= K and over the gate
        eng.set_quantize_limit(*lim)
        got = eng.process_frames(imgs, deps, op, sm.sig_ids, n_total, vp)
        for a, b in zip(base[:4], got[:4]):
            assert np.array_equal(a, b), lim
        for a, b in zip(base[4], got[4]):
            assert a["ok"] == b["ok"] and a["n_matches"] == b["n_matches"] and a["n_inliers"] == b["n_inliers"]
            assert np.array_equal(a["rvec"], b["rvec"]) and np.array_equal(a["tvec"], b["tvec"])


def test_bad_signature_gate_at_the_threshold(world):
    """two frames of one batch, threshold - 1 and threshold keypoints: the first is a bad signature, the second is quantised"""
    sm = world.smap
    n_total = len(sm.sig_ids) + 1
    g = grid_image(step=40)
    dep_b = np.full(g.shape, 1000, np.uint16)
    op = Engine.orb_params(K4, n_features=DET)
    det = engine(DETECTOR_GFTT_ORB, min_distance=0.0)
    kp_b, d_b, _ = det.orb_detect_describe(g[None], dep_b[None], op, cap=DET)[0]
    n = len(kp_b)
    assert 20 < n < DET
    weakest = int(np.argmin(np.abs(kp_b[:, 4]) + (np.arange(n) == 0)))  # any corner that is not alone at the maximum
    dep_a = dep_b.copy()
    dep_a[int(kp_b[weakest, 1]), int(kp_b[weakest, 0])] = 0
    kp_a = det.orb_detect_describe(g[None], dep_a[None], op, cap=DET)[0][0]
    assert len(kp_a) == n - 1
    eng = load(engine(DETECTOR_GFTT_ORB, min_distance=0.0), world)
    eng.set_quantize_limit(n // 2, 1.0, n)   # threshold int(1.0f * n) = n
    vp = Engine.verify_params(K4)
    imgs = np.stack([g, g])
    nkp, words, like, hyp, res = eng.process_frames(imgs, np.stack([dep_a, dep_b]), op, sm.sig_ids, n_total, vp)
    assert nkp.tolist() == [n - 1, n]
    assert words[0][:n - 1].tolist() == [-(i + 1) for i in range(n - 1)] and (words[0][n - 1:] == 0).all()
    assert (like[0] == 0).all() and hyp[0] == 0 and not res[0]["ok"] and res[0]["n_matches"] == 0
    w_o, l_o = expected(oracle_dict(world), kp_b, d_b, sm.sig_ids, n_total, n // 2, 1.0, n)
    assert (w_o > 0).sum() == n // 2
    assert np.array_equal(words[1][:n], w_o) and np.allclose(like[1], l_o, atol=1e-4, rtol=1e-4)
    assert hyp[1] == top(l_o, sm.sig_ids)[0]


def test_map_frame_with_the_limit_equals_the_per_call_sequence():
    """lcd_map_frame under the limit = detect + update + quantise the picked rows + ni := keypoint count + score; a bad frame adds no
    words and no references"""
    rng = np.random.default_rng(3)
    op = Engine.orb_params(K4, n_features=DET)
    base = [(synth.make_image(480, 640, 700 + p, bgr=True), synth.make_depth(480, 640, 750 + p)) for p in range(3)]
    frames = [synth.render_view(*base[t % 3], int(rng.integers(-4, 5)), int(rng.integers(-4, 5)), 2.0, rng) for t in range(6)]
    sparse = np.repeat(grid_image(step=120)[..., None], 3, axis=2)                 # a few corners: under the gate
    frames.insert(4, (sparse, np.full(sparse.shape[:2], 1000, np.uint16)))
    pipe, seq = engine(), engine()
    pipe.set_quantize_limit(K, 0.5, K)
    saw_bad = saw_cut = False
    for t, (img, dep) in enumerate(frames):
        sig = t + 1
        wm = np.arange(1, sig, dtype=np.int32)
        size0 = pipe.size
        pipe.map_detect_async(img, dep, op)
        n_kp, words, n_new, like = pipe.map_frame(sig, wm, sig)
        kp, d, _ = seq.orb_detect_describe(img[None], dep[None], op, cap=DET)[0]
        seq.update()
        created = []

        def quantize(raw):
            w, nn = seq.quantize(d[raw], sig)
            created.append(nn)
            return w

        w_o, raw = lk.signature_word_ids(kp, K, 0.5, K, quantize)
        seq.set_ni([sig], [len(kp)])
        assert n_kp == len(kp) and np.array_equal(words, w_o), t
        assert n_new == (created[0] if created else 0)
        if not created:
            saw_bad = True
            assert n_new == 0 and (words < 0).all() and pipe.size == size0
        saw_cut |= len(kp) > K
        if len(wm):
            l_o = seq.score(w_o, wm, sig)
            assert like is not None and np.allclose(like, l_o, atol=1e-6, rtol=1e-6)
        for w in np.unique(words[words > 0]):
            a, b = pipe.get_refs(int(w)), seq.get_refs(int(w))
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert saw_bad and saw_cut
    assert pipe.total_refs() == seq.total_refs()


def test_sharded_step_with_the_limit_equals_the_unsharded_call(world):
    import torch

    sm = world.smap
    ns = len(sm.sig_ids)
    eng = load(engine(), world)
    eng.set_quantize_limit(K, 0.5, K)
    imgs, deps, _ = synth.make_view_frames(world, 5, seed=4)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    nf = len(imgs)
    d_img = torch.from_numpy(imgs).cuda()
    d_dep = torch.from_numpy(deps.view(np.int16)).cuda()
    d_sig = torch.from_numpy(sm.sig_ids).cuda()
    d_rowids = torch.from_numpy(world.word_ids).cuda()
    ext = torch.cuda.ExternalStream(eng.stream)
    with torch.cuda.stream(ext):
        w0 = torch.zeros(nf * DET, dtype=torch.int32, device="cuda")
        l0 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        eng.process_frames_dev(d_img.data_ptr(), nf, 640, 480, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, ns + 1, vp, w0.data_ptr(), l0.data_ptr())
        hyp0, res0 = eng.process_fetch(nf)
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        w1 = torch.zeros(nf * DET, dtype=torch.int32, device="cuda")
        l1 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        for _ in range(2):
            eng.shard_process_frames_dev(d_img.data_ptr(), nf, 640, 480, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, ns + 1, d_rowids.data_ptr(),
                                         int(world.word_ids.max()), vp, w1.data_ptr(), l1.data_ptr(), True, 0.8, True)
        hyp1, res1 = eng.process_fetch(nf)
        eng.shard_comm_destroy()
    w0n = w0.cpu().numpy()
    assert (w0n < 0).any() and torch.equal(w0, w1) and torch.equal(l0, l1)
    assert np.array_equal(hyp0, hyp1) and (hyp0 > 0).all()
    for a, b in zip(res0, res1):
        assert a["ok"] == b["ok"] and a["n_inliers"] == b["n_inliers"] and np.array_equal(a["rvec"], b["rvec"])


def _limit_dev(eng, kp, n, desc):
    """lcd_limit_keypoints_dev on host arrays: kp [F, cap] KP_DTYPE, n [F], desc [F, cap, row] -> (desc_out, index, n_q)"""
    import torch

    F, cap = kp.shape
    k = eng.quantize_limit[0]
    k = min(k, cap) if k > 0 else cap
    d_kp = torch.from_numpy(kp.view(np.uint8).copy()).cuda()
    d_n = torch.from_numpy(np.asarray(n, np.int32)).cuda()
    d_desc = torch.from_numpy(desc).cuda()
    d_out = torch.full((F, k) + desc.shape[2:], 7, dtype=d_desc.dtype, device="cuda")
    d_idx = torch.full((F, k), 7, dtype=torch.int32, device="cuda")
    d_nq = torch.full((F,), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.limit_keypoints_dev(F, cap, d_kp.data_ptr(), d_n.data_ptr(), d_desc.data_ptr(), d_out.data_ptr(), d_idx.data_ptr(), d_nq.data_ptr())
    eng.synchronize()
    return d_out.cpu().numpy(), d_idx.cpu().numpy(), d_nq.cpu().numpy()


@pytest.mark.parametrize("kind", ["binary", "float64"])
def test_limit_keypoints_dev_against_the_oracle(kind):
    rng = np.random.default_rng(17)
    cap = 4096
    eng = Engine() if kind == "binary" else Engine(desc_type=LCD_DESC_F32, desc_dim=64)
    counts = [4096, 0, 4096, 3000, 1, 2049]
    F = len(counts)
    kp = np.zeros((F, cap), KP_DTYPE)
    kp["response"] = (rng.integers(0, 40, (F, cap)) * rng.choice([-1, 1], (F, cap))).astype(np.float32) * np.float32(1e-4)
    kp["response"][:, ::97] = -0.0
    kp["x"] = rng.uniform(0, 640, (F, cap))
    desc = rng.integers(0, 256, (F, cap, 32), dtype=np.uint8) if kind == "binary" else rng.normal(0, 1, (F, cap, 64)).astype(np.float32)
    for lim in ((1, 0.0, 0), (4095, 0.0, 0), (5000, 0.0, 0), (0, 0.0, 0), (1000, 0.5, 5000)):   # gate 2500: frames 4 and 5 fail it
        eng.set_quantize_limit(*lim)
        out, idx, nq = _limit_dev(eng, kp, counts, desc)
        k = out.shape[1]
        thr = lk.bad_sign_threshold(lim[1], lim[2])
        for f, n in enumerate(counts):
            r = kp["response"][f, :n]
            raw = np.flatnonzero(lk.limit_keypoints_inliers(r, lim[0])) if n and n >= thr else np.zeros(0, np.int64)
            q = len(raw)
            assert nq[f] == q, (lim, f)
            assert np.array_equal(idx[f, :q], raw) and (idx[f, q:] == -1).all(), (lim, f)
            assert np.array_equal(out[f, :q], desc[f, raw]) and (out[f, q:] == 0).all(), (lim, f)
        # batch position: the frames reversed give each frame the same rows
        out2, idx2, nq2 = _limit_dev(eng, kp[::-1].copy(), counts[::-1], desc[::-1].copy())
        assert np.array_equal(out2[::-1], out) and np.array_equal(idx2[::-1], idx) and np.array_equal(nq2[::-1], nq)


def test_word_ids_expand_dev_numbers_the_other_rows():
    import torch

    rng = np.random.default_rng(4)
    eng = Engine()
    cap, k = 4096, 1000
    counts = np.array([4096, 0, 1500, 999, 3], np.int32)
    F = len(counts)
    idx = np.full((F, k), -1, np.int32)
    nq = np.zeros(F, np.int32)
    for f, n in enumerate(counts):
        q = min(k, n) if f != 3 else 0      # frame 3: a bad signature
        idx[f, :q] = np.sort(rng.choice(n, q, replace=False)) if q else []
        nq[f] = q
    wq = rng.integers(1, 50000, (F, k)).astype(np.int32)
    dn, di, dq, dw = (torch.from_numpy(a).cuda() for a in (counts, idx, nq, wq))
    out = torch.full((F, cap), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.word_ids_expand_dev(F, cap, k, dn.data_ptr(), di.data_ptr(), dq.data_ptr(), dw.data_ptr(), out.data_ptr())
    eng.synchronize()
    got = out.cpu().numpy()
    for f, n in enumerate(counts):
        q = nq[f]
        want = np.zeros(cap, np.int32)
        picked = np.zeros(n, bool)
        picked[idx[f, :q]] = True
        want[idx[f, :q]] = wq[f, :q]
        want[np.flatnonzero(~picked)] = -np.arange(1, n - q + 1)
        assert np.array_equal(got[f], want), f


def test_device_decision_chain_equals_the_host_split(world):
    """detect -> lcd_limit_keypoints_dev -> localize -> decide -> lcd_word_ids_expand_dev -> epipolar check on the full uv -> verification
    on the full rows, all on the device, equals the same chain with the limit and the expansion computed on the host"""
    import torch
    from bayes_cases import PATTERNS, make_graph, n_levels, with_vp
    from oracle.bayes_py import parse_prediction_lc, prediction_columns

    sm = world.smap
    places = [int(s) for s in sm.sig_ids]
    ns, B = len(places), 4
    tables, stm = make_graph("chain", places, n_levels(PATTERNS["default"]), np.random.default_rng(1))
    ids = with_vp(places, True)
    cp, rows, lv = prediction_columns(ids, tables.__getitem__, stm)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    det = engine()
    place_kp = [det.orb_detect_describe(world.images[p][None], world.depths[p][None], op, cap=DET)[0][0] for p in range(len(world.images))]
    uv_store = np.zeros((ns, DET, 2), np.float32)
    for i, p in enumerate(world.sig_place):
        kpp = place_kp[int(p)]
        uv_store[i, :len(kpp)] = kpp[:, :2]
    imgs, deps, _ = synth.make_view_frames(world, B, seed=6, max_shift=4)
    d_img = torch.from_numpy(imgs).cuda()
    d_dep = torch.from_numpy(deps.view(np.int16)).cuda()
    d_sig = torch.from_numpy(sm.sig_ids).cuda()
    outs = []
    for on_device in (True, False):
        eng = load(engine(), world)
        eng.sig_words_add_batch(sm.sig_ids, sm.sig_words, uv_store, sm.ni)
        eng.clients_create(B)
        eng.clients_set_map(ids, cp, rows, lv, parse_prediction_lc(PATTERNS["default"]), 0.9)
        eng.set_quantize_limit(K, 0.5, K)
        d_kp = torch.zeros((B, DET, 24), dtype=torch.uint8, device="cuda")
        d_desc = torch.zeros((B, DET, 32), dtype=torch.uint8, device="cuda")
        d_uv = torch.zeros((B, DET, 2), dtype=torch.float32, device="cuda")
        d_xyz = torch.zeros((B, DET, 3), dtype=torch.float32, device="cuda")
        d_n = torch.zeros(B, dtype=torch.int32, device="cuda")
        d_q = torch.zeros((B, K, 32), dtype=torch.uint8, device="cuda")
        d_idx = torch.zeros((B, K), dtype=torch.int32, device="cuda")
        d_nq = torch.zeros(B, dtype=torch.int32, device="cuda")
        d_wq = torch.zeros((B, K), dtype=torch.int32, device="cuda")
        d_w = torch.zeros((B, DET), dtype=torch.int32, device="cuda")
        d_like = torch.zeros((B, ns), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        eng._check(eng._lib.lcd_orb_detect_describe_dev(eng.handle, B, d_img.data_ptr(), 640, 480, 3, d_dep.data_ptr(), 1, ctypes.byref(op),
                                                        DET, d_kp.data_ptr(), d_desc.data_ptr(), d_xyz.data_ptr(), d_uv.data_ptr(), d_n.data_ptr(), None))
        eng.synchronize()
        if on_device:
            eng.limit_keypoints_dev(B, DET, d_kp.data_ptr(), d_n.data_ptr(), d_desc.data_ptr(), d_q.data_ptr(), d_idx.data_ptr(), d_nq.data_ptr())
        else:
            kp = d_kp.cpu().numpy().reshape(-1).view(KP_DTYPE).reshape(B, DET)
            n = d_n.cpu().numpy()
            desc = d_desc.cpu().numpy()
            q = np.zeros((B, K, 32), np.uint8)
            for f in range(B):
                raw = np.flatnonzero(lk.limit_keypoints_inliers(kp["response"][f, :n[f]], K))
                assert len(raw) == K
                q[f] = desc[f, raw]
                d_idx[f] = torch.from_numpy(raw.astype(np.int32))
            d_q.copy_(torch.from_numpy(q))
            d_nq.fill_(K)
        torch.cuda.synchronize()
        eng.localize_batch_dev(d_q.data_ptr(), B, K, d_sig.data_ptr(), ns, ns + 1, d_wq.data_ptr(), d_like.data_ptr())
        eng.synchronize()
        eng.decide_batch_dev(d_like.data_ptr(), B, ns, list(range(B)), [0] * B, Engine.decide_params())
        if on_device:
            eng.word_ids_expand_dev(B, DET, K, d_n.data_ptr(), d_idx.data_ptr(), d_nq.data_ptr(), d_wq.data_ptr(), d_w.data_ptr())
        else:
            n = d_n.cpu().numpy()
            wq = d_wq.cpu().numpy()
            idx = d_idx.cpu().numpy()
            w = np.zeros((B, DET), np.int32)
            for f in range(B):
                picked = np.zeros(n[f], bool)
                picked[idx[f]] = True
                w[f, np.flatnonzero(~picked)] = -np.arange(1, n[f] - K + 1)
                w[f, idx[f]] = wq[f]
            d_w.copy_(torch.from_numpy(w))
        torch.cuda.synchronize()
        eng.decide_epipolar_dev(d_w.data_ptr(), d_uv.data_ptr(), d_n.data_ptr(), B, DET)
        eng.verify_decided_dev(d_desc.data_ptr(), d_uv.data_ptr(), B, DET, vp)
        hyp, res = eng.process_fetch(B)
        outs.append((d_w.cpu().numpy(), d_like.cpu().numpy(), eng.decide_fetch(B), eng.epipolar_fetch(B), hyp, res, d_n.cpu().numpy()))
    a, b = outs
    assert (a[6] > K).all()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and np.array_equal(a[4], b[4])
    assert (a[0] < 0).any()
    for x, y in zip(a[3], b[3]):
        assert x["checked"] == y["checked"] and x["ok"] == y["ok"] and x["n_pairs"] == y["n_pairs"] and x["n_inliers"] == y["n_inliers"]
    for x, y in zip(a[5], b[5]):
        assert x["ok"] == y["ok"] and x["n_matches"] == y["n_matches"] and x["n_inliers"] == y["n_inliers"]
    assert any(x["checked"] for x in a[3])


def test_refusals_keep_the_previous_setting():
    eng = Engine()
    eng.set_quantize_limit(300, 0.5, 400)
    for bad in ((-1, 0.5, 400), (300, -0.1, 400), (300, float("nan"), 400), (300, float("inf"), 400), (300, 0.5, -2)):
        with pytest.raises(LcdError) as ex:
            eng.set_quantize_limit(*bad)
        assert ex.value.code == -1
        assert eng.quantize_limit == (300, 0.5, 400)
    eng._check(eng._lib.lcd_quantize_limit_set(eng.handle, None))
    assert eng.quantize_limit == (0, 0.0, 0)
    with pytest.raises(LcdError):
        eng.word_ids_expand_dev(1, 100, 101, 1, 1, 1, 1, 1)
    with pytest.raises(LcdError):
        eng.limit_keypoints_dev(1, 4097, 1, 1, 1, 1, 1, 1)
