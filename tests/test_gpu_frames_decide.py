"""lcd_process_frames_decide_submit / _dev: Rtabmap::process's localisation step from images for many clients in one call.  Engine A runs
the new call; engine B holds the same map and runs the public composition (lcd_process_frames for words and likelihood, the decision
calls on its likelihood rows, lcd_verify_batch on each frame's own detected rows for every registration).  Over many steps with a
repeating client pattern, so the posteriors carry state, every output must agree bit for bit."""
import numpy as np
import pytest

from oracle import decide_py as dc
from rtabmap_b200 import Engine, LcdError, synth
from rtabmap_b200.capi import (DECISION_DTYPE, DETECTOR_GFTT_ORB, DETECTOR_ORB, DETECTOR_ORB_OCTREE, EpipolarParams, EpipolarResult,
                               ProximityResult, VerifyResult)

pytestmark = pytest.mark.gpu

K4 = synth.CAMERA_K4
DET, K = 600, 300
B, N_CLIENTS, STEPS = 6, 9, 10
H, W = 480, 640
ACCEPTED, VERIFY_REJECTED, EPIPOLAR_REJECTED, PROXIMITY_SUPPRESSED = 8, 9, 11, 12


def engine(detector):
    e = Engine(max_words=16384, max_signatures=400)
    if detector == DETECTOR_GFTT_ORB:
        e.set_detector(DETECTOR_GFTT_ORB, Engine.gftt_params())
    elif detector == DETECTOR_ORB_OCTREE:
        e.set_detector_orb_octree()
    return e


_WORLDS = {}


def world(detector):
    if detector not in _WORLDS:
        det = engine(detector)
        op = Engine.orb_params(K4, n_features=DET)
        w = synth.make_place_world(lambda im, dp: det.orb_detect_describe(im[None], dp[None], op, cap=DET)[0], 4, 3000, 24, DET, H, W, seed=11)
        kps = [det.orb_detect_describe(w.images[p][None], w.depths[p][None], op, cap=DET)[0][0] for p in range(len(w.images))]
        _WORLDS[detector] = (w, kps)
    return _WORLDS[detector]


def pose_at(x, y=0.0):
    p = np.zeros((3, 4), np.float32)
    p[:, :3] = np.eye(3, dtype=np.float32)
    p[0, 3], p[1, 3] = x, y
    return p


def sig_x(i):
    """x of signature row i (a view of place i % 4): each place's six views 0.3 m apart, places 2 m apart, so the views of a frame's own
    place, and only those, lie within its proximity radius"""
    return 2.0 * (i % 4) + 0.3 * (i // 4)


def gps_at(x, stamp=1.0):
    return (stamp, -73.6 + 1.28e-5 * x, 45.5, 30.0, 2.0)   # about 1 m of longitude per metre of x


def map_arrays(detector):
    """the stores the map is loaded with.  Some views are made to fail on purpose: views 1 and 3 of each place have no 3-D points (their
    registration fails: LCD_DECIDE_VERIFY_REJECTED, or LCD_DECIDE_PROXIMITY_SUPPRESSED when proximity registers another view), view 4 has
    no words in the word store (0 epipolar pairs: LCD_DECIDE_EPIPOLAR_REJECTED)"""
    w, kps = world(detector)
    sm = w.smap
    view = np.arange(len(sm.sig_ids)) // 4
    xyz = w.store.xyz.copy()
    xyz[np.isin(view, (1, 3))] = np.nan
    n_words = np.where(view == 4, 0, sm.ni).astype(np.int32)
    uv = np.zeros((len(sm.sig_ids), DET, 2), np.float32)
    for i, p in enumerate(w.sig_place):
        uv[i, :len(kps[int(p)])] = kps[int(p)][:, :2]
    return w.store.desc, xyz, n_words, uv


def load(detector):
    """one engine holding the world's map: dictionary, index, stores, Bayes map, poses and GPS"""
    from bayes_cases import PATTERNS, make_graph, n_levels, with_vp
    from oracle.bayes_py import parse_prediction_lc, prediction_columns

    w, kps = world(detector)
    sm = w.smap
    places = [int(s) for s in sm.sig_ids]
    e = engine(detector)
    e.add_words(w.word_ids, w.vocab)
    e.last_word_id = int(w.word_ids.max())
    e.update()
    e.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    e.set_ni(sm.sig_ids, sm.ni)
    desc, xyz, n_words, uv = map_arrays(detector)
    e.sig_add_batch(sm.sig_ids, desc, xyz, sm.ni)
    e.sig_words_add_batch(sm.sig_ids, sm.sig_words, uv, n_words)
    e.clients_create(N_CLIENTS)
    tables, stm = make_graph("chain", places, n_levels(PATTERNS["default"]), np.random.default_rng(1))
    ids = with_vp(places, True)
    cp, rows, lv = prediction_columns(ids, tables.__getitem__, stm)
    e.clients_set_map(ids, cp, rows, lv, parse_prediction_lc(PATTERNS["default"]), 0.9)
    ptr = np.concatenate([[0], np.cumsum([(i > 0) + (i + 1 < len(places)) for i in range(len(places))])]).astype(np.int64)
    nbr = np.array([places[j] for i in range(len(places)) for j in (i - 1, i + 1) if 0 <= j < len(places)], np.int32)
    e.clients_set_map_poses(places, np.stack([pose_at(sig_x(i)) for i in range(len(places))]), ptr, nbr)
    gps = np.array([gps_at(sig_x(i)) for i in range(len(places))])
    gps[::5, 0] = 0.0  # places without a fix are always compared
    e.clients_set_map_gps(places, gps)
    return e, places


def frames(detector, step):
    """B frames of step `step`: revisits, one all-black frame (no keypoint) and one short frame (a small textured patch: few keypoints,
    the rest of its rows padding)"""
    w, _ = world(detector)
    imgs, deps, places = synth.make_view_frames(w, B, seed=100 + step, max_shift=4)
    places = places.copy()
    if step % 3 == 1:
        imgs[1] = 0
        places[1] = -1
    if step % 3 == 2:
        short = np.zeros_like(imgs[2])
        short[200:270, 290:380] = imgs[2][200:270, 290:380]
        imgs[2] = short
    return np.ascontiguousarray(imgs), np.ascontiguousarray(deps), places


def step_inputs(step, n_places, places):
    clients = np.array([(3 * step + f) % N_CLIENTS for f in range(B)], np.int32)   # a repeating pattern: state carries over
    flags = np.zeros(B, np.int32)
    if step % 4 == 3:
        flags[3] = dc.FRAME_HOLD
    if step % 5 == 4:
        flags[4] = dc.FRAME_SKIP
    flags[::2] |= dc.FRAME_AGGRESSIVE
    x = 2.0 * np.where(places >= 0, places, 0) + 0.75          # amid the views of the frame's place
    gps = np.array([gps_at(v) for v in x])
    gps[::3, 0] = 0.0
    poses = np.stack([pose_at(v, 0.05) for v in x])
    enabled = np.ones(B, np.int32)
    enabled[5] = 0
    return clients, flags, gps, poses, enabled


def detected(eng, imgs, deps, op):
    """lcd_orb_detect_describe's rows of each frame, zero-padded to DET: descriptors, 3-D points and keypoints"""
    desc = np.zeros((B, DET, 32), np.uint8)
    xyz = np.zeros((B, DET, 3), np.float32)
    uv = np.zeros((B, DET, 2), np.float32)
    for f, (k, d, x) in enumerate(eng.orb_detect_describe(imgs, deps, op, cap=DET)):
        desc[f, :len(d)], xyz[f, :len(d)], uv[f, :len(d)] = d, x, k[:, :2]
    return desc, xyz, uv


def verify_own_rows(eng, slot_ids, store, sig_ids, desc, xyz, uv, n_kp, vp):
    """lcd_verify_batch of (stored place, frame) pairs with TO = the frame's own n_kp rows, their uv and xyz"""
    row = {int(s): i for i, s in enumerate(sig_ids)}
    fr = [row[int(s)] for s, _ in slot_ids]
    fi = [f for _, f in slot_ids]
    n_from = np.array([store.n[r] for r in fr], np.int32)
    res = eng.verify_batch(store.desc[fr], store.xyz[fr], desc[fi], uv[fi], K4, n_from=n_from, n_to=n_kp[fi], xyz_to=xyz[fi],
                           min_inliers=vp.min_inliers)
    return res[0] if isinstance(res, tuple) else res


def same(a, b, where):
    """a: a registration as the decision calls report it, b: lcd_verify_batch's"""
    assert (a["ok"], a["n_matches"], a["n_inliers"], a["iterations_run"]) == (b["ok"], len(b["matches"]), len(b["inliers"]), b["iterations_run"]), where
    for k in ("rvec", "tvec", "transform", "covariance"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), f"{where}: {k}"


STAGES = ("none", "gps", "all")
GPS_RADIUS = 5.0   # RGBD/LocalRadius of the GPS filter: a frame compares its own place and its neighbours'



@pytest.mark.parametrize("detector", [DETECTOR_ORB, DETECTOR_GFTT_ORB, DETECTOR_ORB_OCTREE])
@pytest.mark.parametrize("limit", [False, True])
@pytest.mark.parametrize("stages", STAGES)
def test_decide_frames_equal_the_composition(detector, limit, stages):
    import torch

    if stages == "gps" and (detector != DETECTOR_ORB or limit):
        pytest.skip("the GPS filter alone is covered once")
    a, places = load(detector)
    b, _ = load(detector)
    ns = len(places)
    w, _ = world(detector)
    store = type("S", (), {})()
    store.desc, store.xyz, _, _ = map_arrays(detector)
    store.n = w.smap.ni
    for e in (a, b):
        if limit:
            e.set_quantize_limit(K, 0.5, 2 * K)   # gate: a frame with fewer than K keypoints is a bad signature
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    dp = Engine.decide_params(loop_thr=0.11)
    ep = EpipolarParams(8, 3.0, 0.99)
    pp = Engine.proximity_params(vp, local_radius=1.2)
    seen = set()
    for step in range(STEPS):
        imgs, deps, fplaces = frames(detector, step)
        clients, flags, gps, poses, enabled = step_inputs(step, ns, fplaces)
        st = Engine.decide_stages(B, frame_gps=gps if stages != "none" else None, local_radius=GPS_RADIUS, epipolar=ep if stages == "all" else None,
                                  proximity=pp if stages == "all" else None, frame_poses=poses, proximity_enabled=enabled)
        # A: the new call
        nkp = np.zeros(B, np.int32)
        words = np.zeros((B, DET), np.int32)
        like = np.zeros((B, ns), np.float32)
        dec = np.zeros(B, DECISION_DTYPE)
        res = (VerifyResult * B)()
        epi = (EpipolarResult * B)()
        prox = (ProximityResult * B)()
        a.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, clients, flags, dp, st, nkp, words, like, dec, res, epi, prox)
        a.process_frames_wait()
        res = Engine._results(res, B)
        # B: the public composition
        nkp_b, words_b, like_b, _, _ = b.process_frames(imgs, deps, op, places, ns + 1, None)
        assert np.array_equal(nkp, nkp_b) and np.array_equal(words, words_b), f"step {step}"
        assert np.array_equal(like.view(np.uint32), like_b.view(np.uint32)), f"step {step}"
        desc, xyz, uv = detected(b, imgs, deps, op)
        bad = np.array([not (words[f, :nkp[f]] > 0).any() for f in range(B)])
        flags_b = flags | np.where(bad, dc.FRAME_SKIP, 0).astype(np.int32)
        d_like = torch.from_numpy(like_b).cuda()
        torch.cuda.synchronize()
        if stages == "none":
            b.decide_batch_dev(d_like.data_ptr(), B, ns, clients, flags_b, dp)
        else:
            b.decide_gps_batch_dev(d_like.data_ptr(), B, ns, clients, flags_b, gps, GPS_RADIUS, dp)
        if stages == "all":
            d_w = torch.from_numpy(words_b).cuda()
            d_uv = torch.from_numpy(uv).cuda()
            d_n = torch.from_numpy(nkp_b).cuda()
            d_q = torch.from_numpy(np.ascontiguousarray(desc)).cuda()
            torch.cuda.synchronize()
            b.decide_epipolar_dev(d_w.data_ptr(), d_uv.data_ptr(), d_n.data_ptr(), B, DET)
            for x, y in zip(Engine.epipolar_records(epi), b.epipolar_fetch(B)):
                assert all(np.array_equal(np.asarray(x[k]), np.asarray(y[k])) for k in x), f"step {step}"
            dec_b = b.decide_fetch(B)
            b.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), B, DET, poses, enabled & ~bad, pp)
            pa, pb = Engine.proximity_records(prox), b.proximity_fetch(B)
            pairs = []
            for f, (x, y) in enumerate(zip(pa, pb)):
                assert (x["status"], x["n_nearest"], x["n_paths"], x["n_attempts"]) == (y["status"], y["n_nearest"], y["n_paths"], y["n_attempts"])
                for p, q in zip(x["paths"], y["paths"]):
                    assert {k: p[k] for k in ("likelihood", "id", "distance", "candidate_id")} == \
                           {k: q[k] for k in ("likelihood", "id", "distance", "candidate_id")}, f"step {step} frame {f}"
                    pairs.append((p["candidate_id"], f, p["result"]))
                seen.add(("prox", x["status"]))
            if pairs:
                want = verify_own_rows(b, [(s, f) for s, f, _ in pairs], store, places, desc, xyz, uv, nkp, vp)
                for (s, f, got), r in zip(pairs, want):
                    same(got, r, f"step {step} proximity {s}/{f}")
        else:
            dec_b = b.decide_fetch(B)
        # decisions: every status before the registrations equal; an accepted frame's registration equals lcd_verify_batch on its own rows
        for f in range(B):
            seen.add(int(dec[f]["status"]))
            assert dec[f]["highest_id"] == dec_b[f]["highest_id"] and dec[f]["highest_value"].view(np.uint32) == dec_b[f]["highest_value"].view(np.uint32)
            if dec_b[f]["status"] != ACCEPTED:
                assert dec[f]["status"] == dec_b[f]["status"] and dec[f]["loop_id"] == dec_b[f]["loop_id"], f"step {step} frame {f}"
                assert not res[f]["ok"] and res[f]["n_matches"] == 0
                continue
            assert dec[f]["status"] in (ACCEPTED, VERIFY_REJECTED, PROXIMITY_SUPPRESSED), f"step {step} frame {f}"
            if stages == "all" and any(p["accepted"] for p in pa[f]["paths"]):
                continue
            r = verify_own_rows(b, [(int(dec_b[f]["loop_id"]), f)], store, places, desc, xyz, uv, nkp, vp)[0]
            same(res[f], r, f"step {step} frame {f}")
            assert dec[f]["status"] == (ACCEPTED if r["ok"] else VERIFY_REJECTED)
        assert all(dec[f]["status"] == 0 and dec[f]["highest_id"] == 0 for f in np.flatnonzero(bad))
        for f in range(B):
            if flags[f] & dc.FRAME_SKIP:
                seen.add("skip flag")
            elif bad[f]:
                seen.add("bad, no keypoint" if nkp[f] == 0 else "bad, gated")   # the gate: keypoints but no quantised word
    want = {ACCEPTED, 1, "skip flag", "bad, no keypoint"}
    if limit:
        want.add("bad, gated")
    if stages == "none":
        want.add(VERIFY_REJECTED)
    if stages == "all":
        want |= {EPIPOLAR_REJECTED, PROXIMITY_SUPPRESSED}
    assert want <= seen, f"not reached: {want - seen} (seen {seen})"


@pytest.mark.parametrize("limit", [False, True])
@pytest.mark.parametrize("stages", ["none", "all"])
def test_posteriors_and_the_oracle(limit, stages):
    """the _dev form: posterior rows bit-equal to the decision call's on the same likelihood, and the decisions equal oracle/decide_py.py's
    restated Rtabmap::process run from the returned likelihood rows (with every optional stage on: up to the registrations)"""
    import torch

    a, places = load(DETECTOR_ORB)
    b, _ = load(DETECTOR_ORB)
    ns = len(places)
    for e in (a, b):
        if limit:
            e.set_quantize_limit(K, 0.5, 2 * K)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    dp = Engine.decide_params()
    oracles = {c: dc.DecideClient() for c in range(N_CLIENTS)}
    for step in range(STEPS):
        imgs, deps, fplaces = frames(DETECTOR_ORB, step)
        clients, flags, gps, poses, enabled = step_inputs(step, ns, fplaces)
        st = None
        if stages == "all":
            st = Engine.decide_stages(B, gps, GPS_RADIUS, EpipolarParams(8, 3.0, 0.99), Engine.proximity_params(vp, local_radius=1.2), poses, enabled)
        d_img = torch.from_numpy(imgs).cuda()
        d_dep = torch.from_numpy(deps.view(np.int16)).cuda()
        d_w = torch.zeros((B, DET), dtype=torch.int32, device="cuda")
        d_l = torch.zeros((B, ns), dtype=torch.float32, device="cuda")
        d_p = torch.full((B, ns + 1), -1.0, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        a.process_frames_decide_dev(d_img.data_ptr(), B, W, H, 3, d_dep.data_ptr(), 1, op, ns, ns + 1, vp, clients, flags, dp, st,
                                    d_w.data_ptr(), d_l.data_ptr(), d_p.data_ptr())
        dec = a.decide_fetch(B)
        words, like = d_w.cpu().numpy(), d_l.cpu().numpy()
        bad = np.array([not (words[f] > 0).any() for f in range(B)])
        flags_b = flags | np.where(bad, dc.FRAME_SKIP, 0).astype(np.int32)
        d_p2 = torch.full((B, ns + 1), -1.0, dtype=torch.float32, device="cuda")
        if st is None:
            b.decide_batch_dev(d_l.data_ptr(), B, ns, clients, flags_b, dp, d_p2.data_ptr())
        else:
            b.decide_gps_batch_dev(d_l.data_ptr(), B, ns, clients, flags_b, gps, GPS_RADIUS, dp, d_p2.data_ptr())
        dec_b = b.decide_fetch(B)
        post, post_b = d_p.cpu().numpy(), d_p2.cpu().numpy()
        assert np.array_equal(post.view(np.uint32), post_b.view(np.uint32)), f"step {step}"
        full = [-1] + places
        for f in range(B):
            assert (dec[f]["highest_id"], dec[f]["highest_value"]) == (dec_b[f]["highest_id"], dec_b[f]["highest_value"])
            if dec_b[f]["status"] != ACCEPTED:
                assert dec[f]["status"] == dec_b[f]["status"]
            want = oracles[int(clients[f])].decide(full, post[f], int(flags_b[f]))
            assert (int(dec[f]["highest_id"]), np.float32(dec[f]["highest_value"])) == (want[0], np.float32(want[1])), f"step {step} frame {f}"
            if want[3] != ACCEPTED:
                assert (int(dec[f]["loop_id"]), int(dec[f]["status"])) == (want[2], want[3]), f"step {step} frame {f}"


def test_pipelined_batches_equal_strict_alternation():
    """batch k+1 submitted before batch k is waited for (one client in both), with a lcd_process_frames_submit batch between two decision
    batches, gives the outputs of strict submit / wait alternation"""
    a, places = load(DETECTOR_ORB)
    b, _ = load(DETECTOR_ORB)
    ns = len(places)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    dp = Engine.decide_params()
    ep = EpipolarParams(8, 3.0, 0.99)
    pp = Engine.proximity_params(vp, local_radius=1.2)
    plan = []
    for step in range(6):
        imgs, deps, fplaces = frames(DETECTOR_ORB, step)
        clients, flags, gps, poses, enabled = step_inputs(step, ns, fplaces)
        plan.append((imgs, deps, clients, flags, Engine.decide_stages(B, gps, GPS_RADIUS, ep, pp, poses, enabled)))
    assert set(plan[0][2]) & set(plan[1][2])

    def outputs():
        return dict(nkp=np.zeros(B, np.int32), words=np.zeros((B, DET), np.int32), like=np.zeros((B, ns), np.float32),
                    dec=np.zeros(B, DECISION_DTYPE), res=(VerifyResult * B)(), epi=(EpipolarResult * B)(), prox=(ProximityResult * B)())

    def submit(e, k, o):
        imgs, deps, clients, flags, st = plan[k]
        e.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, clients, flags, dp, st, o["nkp"], o["words"], o["like"], o["dec"], o["res"],
                                       o["epi"], o["prox"])

    def plain(e, k, o):
        imgs, deps = plan[k][:2]
        e.process_frames_submit(imgs, deps, op, np.array(places, np.int32), ns + 1, vp, o["nkp"], o["words"], o["like"], np.zeros(B, np.int32), o["res"])

    def flat(o):
        return [o["nkp"].tobytes(), o["words"].tobytes(), o["like"].tobytes(), o["dec"].tobytes(), bytes(o["res"]), bytes(o["epi"]), bytes(o["prox"])]

    strict, piped = [], []
    kinds = [submit, submit, plain, submit, submit, submit]
    for k, fn in enumerate(kinds):
        o = outputs()
        fn(b, k, o)
        b.process_frames_wait()
        strict.append(flat(o))
    outs = [outputs() for _ in kinds]
    kinds[0](a, 0, outs[0])
    for k in range(1, len(kinds)):
        kinds[k](a, k, outs[k])      # two batches in flight
        with pytest.raises(LcdError):
            submit(a, 0, outputs())  # a third is refused
        a.process_frames_wait()
    a.process_frames_wait()
    for k in range(len(kinds)):
        got = flat(outs[k])
        for i, (x, y) in enumerate(zip(got, strict[k])):
            assert x == y, f"batch {k} output {i}"


def test_refusals_change_nothing():
    """each refusal returns its code, and the next step gives what it gives when the refused call was never made"""
    ref, places = load(DETECTOR_ORB)
    ns = len(places)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    dp = Engine.decide_params()
    imgs, deps, fplaces = frames(DETECTOR_ORB, 0)
    clients, flags, gps, poses, enabled = step_inputs(0, ns, fplaces)

    def run(e):
        d = np.zeros(B, DECISION_DTYPE)
        like = np.zeros((B, ns), np.float32)
        e.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, clients, flags, dp, None, None, None, like, d)
        e.process_frames_wait()
        return d.tobytes(), like.tobytes()

    def code(f):
        with pytest.raises(LcdError) as ex:
            f()
        return ex.value.code

    want = [run(ref), run(ref)]
    e, _ = load(DETECTOR_ORB)
    sub = lambda **kw: e.process_frames_decide_submit(imgs, deps, kw.get("op", op), kw.get("ns", ns), ns + 1, vp, kw.get("clients", clients),
                                                      kw.get("flags", flags), kw.get("dp", dp), kw.get("st"))
    assert code(lambda: sub(clients=np.array([0, 0, 1, 2, 3, 4]))) == -1                      # a client listed twice
    assert code(lambda: sub(ns=ns - 1)) == -1                                                  # not the map's places
    assert code(lambda: sub(dp=Engine.decide_params(loop_thr=2.0))) == -1                      # bad parameters
    assert code(lambda: sub(op=Engine.orb_params(K4, n_features=0))) == -3
    assert code(lambda: sub(st=Engine.decide_stages(B, local_radius=-1.0, frame_gps=gps))) == -1
    assert code(lambda: sub(st=Engine.decide_stages(B, proximity=Engine.proximity_params(vp, max_paths=0), frame_poses=poses,
                                                    proximity_enabled=enabled))) == -3
    bad = poses.copy()
    bad[0, 0, 3] = np.nan
    assert code(lambda: sub(st=Engine.decide_stages(B, proximity=Engine.proximity_params(vp), frame_poses=bad, proximity_enabled=enabled))) == -1
    assert run(e) == want[0]
    # no GPS table / no poses for the current map / no clients / no map: LCD_ERR_STATE
    from bayes_cases import PATTERNS, make_graph, n_levels, with_vp
    from oracle.bayes_py import parse_prediction_lc, prediction_columns

    tables, stm = make_graph("chain", places, n_levels(PATTERNS["default"]), np.random.default_rng(1))
    ids = with_vp(places, True)
    cp, rows, lv = prediction_columns(ids, tables.__getitem__, stm)
    e.clients_set_map(ids, cp, rows, lv, parse_prediction_lc(PATTERNS["default"]), 0.9)   # the same map again: no GPS table, no poses
    assert code(lambda: sub(st=Engine.decide_stages(B, frame_gps=gps))) == -4
    assert code(lambda: sub(st=Engine.decide_stages(B, proximity=Engine.proximity_params(vp), frame_poses=poses, proximity_enabled=enabled))) == -4
    assert run(e) == want[1]
    fresh = engine(DETECTOR_ORB)
    fresh.add_words(world(DETECTOR_ORB)[0].word_ids[:10], world(DETECTOR_ORB)[0].vocab[:10])
    fresh.update()
    fresh.sig_add_batch([1], world(DETECTOR_ORB)[0].store.desc[:1], world(DETECTOR_ORB)[0].store.xyz[:1], [5])
    assert code(lambda: fresh.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, clients, flags, dp)) == -4   # no clients
    fresh.clients_create(N_CLIENTS)
    assert code(lambda: fresh.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, clients, flags, dp)) == -4   # no map
    f32 = Engine(desc_type=1, desc_dim=64, max_words=64)
    assert code(lambda: f32.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, clients, flags, dp)) == -1
    sharded, _ = load(DETECTOR_ORB)
    sharded.shard_set_row_offset(5)
    assert code(lambda: sharded.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, clients, flags, dp)) == -4


@pytest.fixture(scope="module")
def map_db(tmp_path_factory):
    """the FAST-ORB world's map written into an RTAB-Map database: each signature's rows in the order the database returns them, neighbour
    links along the signature ids, optimised poses and a GPS fix on every node"""
    from test_dbio_map import make_map_db, relative

    from rtabmap_b200 import dbio, graph

    w, _ = world(DETECTOR_ORB)
    sm = w.smap
    S, F = sm.sig_words.shape
    ids = [int(s) for s in sm.sig_ids]
    desc, xyz, _, uv = map_arrays(DETECTOR_ORB)
    order = np.stack([np.argsort(np.where(np.arange(F) < sm.ni[k], sm.sig_words[k], np.iinfo(np.int32).max), kind="stable") for k in range(S)])
    words = np.take_along_axis(sm.sig_words, order, 1)
    desc = np.take_along_axis(desc, order[:, :, None], 1)
    xyz = np.take_along_axis(xyz, order[:, :, None], 1)
    uv = np.take_along_axis(uv, order[:, :, None], 1)
    fin = np.isfinite(xyz).all(2)
    poses = {s: pose_at(sig_x(k)) for k, s in enumerate(ids)}
    links = []
    for a, b in zip(ids[:-1], ids[1:]):
        links += [(a, b, graph.NEIGHBOR, relative(poses[a], poses[b])), (b, a, graph.NEIGHBOR, relative(poses[b], poses[a]))]
    gps = {s: gps_at(sig_x(k), 1000.0 + s) + (0.0,) for k, s in enumerate(ids)}
    feats = [(s, int(words[k, j]), uv[k, j, 0], uv[k, j, 1], xyz[k, j] if fin[k, j] else None, desc[k, j].tobytes())
             for k, s in enumerate(ids) for j in range(int(sm.ni[k]))]
    db = str(tmp_path_factory.mktemp("db") / "map.db")
    make_map_db(db, w.word_ids, w.vocab, ids, feats, links, (np.array(ids, np.int32), np.stack([poses[s] for s in ids])), gps, poses=poses)
    ln = dbio.Links(np.array([l[0] for l in links], np.int32), np.array([l[1] for l in links], np.int32), np.array([l[2] for l in links], np.int32),
                    np.stack([l[3] for l in links]))
    o = np.lexsort((ln.to_id, ln.from_id))
    ln = dbio.Links(ln.from_id[o], ln.to_id[o], ln.type[o], ln.transform[o])
    return dict(db=db, ids=ids, words=words, desc=desc, xyz=xyz, uv=uv, links=ln, poses=poses, gps=gps)


def test_a_map_opened_from_a_database_serves_the_call(map_db):
    """dbio.open_localization_map's engine answers the call, stages and all, bit for bit as an engine set up by hand from the same arrays"""
    from rtabmap_b200 import dbio, graph

    M = map_db
    ids = M["ids"]
    ns = len(ids)
    w, _ = world(DETECTOR_ORB)
    sm = w.smap
    loaded = engine(DETECTOR_ORB)
    loaded.clients_create(N_CLIENTS)
    r = dbio.open_localization_map(loaded, M["db"])
    assert list(r.places) == ids and r.poses_set and r.gps_set and set(r.skipped) == {"global_descriptors"}   # none were written
    hand = engine(DETECTOR_ORB)
    hand.add_words(w.word_ids, w.vocab)
    hand.last_word_id = int(w.word_ids.max())
    hand.update()
    hand.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    hand.set_ni(sm.sig_ids, sm.ni)
    hand.sig_add_batch(ids, M["desc"], M["xyz"], sm.ni)
    hand.sig_words_add_batch(ids, M["words"], M["uv"], sm.ni)
    hand.clients_create(N_CLIENTS)
    lc = graph.DEFAULT_PREDICTION_LC
    tab = graph.prediction_tables(ids, graph.bayes_neighbors(ids, M["links"], len(lc) - 1))
    hand.clients_set_map(tab[0], tab[1], tab[2], tab[3], lc, 0.9)
    pose = np.stack([M["poses"][s] for s in ids])
    hand.clients_set_map_poses(ids, pose, *graph.neighbor_links(ids, M["links"]))
    g6 = np.array([M["gps"][s] for s in ids], np.float64)
    gps, off = graph.gps_of_places(ids, g6, pose, M["links"])
    hand.clients_set_map_gps(ids, gps[:, :5], off)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    dp = Engine.decide_params()
    statuses = set()
    for step in range(4):
        imgs, deps, fplaces = frames(DETECTOR_ORB, step)
        clients, flags, fgps, poses, enabled = step_inputs(step, ns, fplaces)
        st = Engine.decide_stages(B, fgps, GPS_RADIUS, EpipolarParams(8, 3.0, 0.99), Engine.proximity_params(vp, local_radius=1.2), poses, enabled)
        got = []
        for e in (loaded, hand):
            o = [np.zeros(B, np.int32), np.zeros((B, DET), np.int32), np.zeros((B, ns), np.float32), np.zeros(B, DECISION_DTYPE),
                 (VerifyResult * B)(), (EpipolarResult * B)(), (ProximityResult * B)()]
            e.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, clients, flags, dp, st, *o)
            e.process_frames_wait()
            got.append([x.tobytes() if isinstance(x, np.ndarray) else bytes(x) for x in o])
            statuses |= {int(s) for s in o[3]["status"]}
        for k, (x, y) in enumerate(zip(*got)):
            assert x == y, f"step {step}: output {k}"
    assert ACCEPTED in statuses, statuses
