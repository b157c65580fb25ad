"""Each localisation client's own camera (lcd_clients_set_cameras) in the decision calls: per-client K through one batched call equals
one call per client with that K, a local transform lifts and registers as the oracle does, the distance checks read the base-frame
transform, clients without a camera are untouched, a batch in flight keeps the cameras it was submitted with, and bad cameras are
refused without a change."""
import ctypes

import numpy as np
import pytest

import camera_oracle as co
from oracle import oracle_py as orc
from rtabmap_b200 import Engine, LcdError, synth
from rtabmap_b200.capi import (DECISION_DTYPE, DETECTOR_ORB, LCD_DESC_F32, EpipolarParams, EpipolarResult, OPTICAL_ROTATION,
                               ProximityResult, VerifyResult, camera_model)
from test_gpu_frames_decide import DET, GPS_RADIUS, H, K4, W, gps_at, load, map_arrays, pose_at, world

pytestmark = pytest.mark.gpu

ACCEPTED, VERIFY_REJECTED, DISTANCE_REJECTED = 8, 9, 10


def ks(n, seed=1):
    """n distinct cameras: fx 480-640, principal point within 20 px of the image centre"""
    rng = np.random.default_rng(seed)
    fx = rng.uniform(480, 640, n)
    return [(float(f), float(f * rng.uniform(0.98, 1.02)), float(320 + rng.uniform(-20, 20)), float(240 + rng.uniform(-20, 20))) for f in fx]


def local_transforms(n, seed=2):
    """the optical rotation after a yaw of the base and an offset of up to 0.5 m"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        a = rng.uniform(-0.3, 0.3)
        L = np.eye(4)
        L[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
        L[:3, 3] = rng.uniform(-0.5, 0.5, 3)
        O = np.eye(4)
        O[:3] = OPTICAL_ROTATION
        out.append((L @ O)[:3].astype(np.float32))
    return out


def view_frames(n, seed):
    w, _ = world(DETECTOR_ORB)
    imgs, deps, places = synth.make_view_frames(w, n, seed=seed, max_shift=4)
    return np.ascontiguousarray(imgs), np.ascontiguousarray(deps), places


def stage_inputs(places):
    n = len(places)
    x = 2.0 * places + 0.75
    gps = np.array([gps_at(v) for v in x])
    gps[::3, 0] = 0.0
    poses = np.stack([pose_at(v, 0.05) for v in x])
    return gps, poses, np.ones(n, np.int32)


class Run:
    """the outputs of one lcd_process_frames_decide_submit batch"""

    def __init__(self, e, imgs, deps, op, ns, vp, clients, dp, st=None, flags=None, wait=True, between=None):
        n = len(imgs)
        self.n = n
        self.nkp = np.zeros(n, np.int32)
        self.words = np.zeros((n, op.n_features), np.int32)
        self.like = np.zeros((n, ns), np.float32)
        self.dec = np.zeros(n, DECISION_DTYPE)
        self.res = (VerifyResult * n)()
        self.epi = (EpipolarResult * n)()
        self.prox = (ProximityResult * n)()
        flags = np.zeros(n, np.int32) if flags is None else flags
        e.process_frames_decide_submit(imgs, deps, op, ns, ns + 1, vp, np.asarray(clients, np.int32), flags, dp, st, self.nkp, self.words,
                                       self.like, self.dec, self.res, self.epi, self.prox)
        if between is not None:
            between()
        if wait:
            e.process_frames_wait()

    def frame(self, f):
        """every output of frame f as bytes"""
        def rec(arr):
            size = ctypes.sizeof(arr) // len(arr)
            return bytes(arr)[f * size:(f + 1) * size]

        return (int(self.nkp[f]), self.words[f].tobytes(), self.like[f].tobytes(), self.dec[f].tobytes(), rec(self.res), rec(self.epi), rec(self.prox))

    def results(self):
        return Engine._results(self.res, self.n)


def with_k(p, K):
    q = type(p).from_buffer_copy(p)
    q.fx, q.fy, q.cx, q.cy = K
    return q


def test_identity_cameras_equal_one_call_per_client():
    """128 clients with their own K and an identity local transform in one batch: every output of every frame is the one-frame call's
    with the client's K in lcd_orb_params and lcd_verify_params"""
    n = 128
    a, places = load(DETECTOR_ORB)
    b, _ = load(DETECTOR_ORB)
    ns = len(places)
    for e in (a, b):
        e.clients_create(n)
    Ks = ks(n)
    a.clients_set_cameras(range(n), [camera_model(k, (W, H)) for k in Ks])
    op = Engine.orb_params(K4, n_features=DET)
    # the frames were rendered with K4: a wider reprojection error lets registrations with the clients' K succeed too
    vp = Engine.verify_params(K4, image_size=(W, H), repeat_once=True, reproj_error=8.0)
    dp = Engine.decide_params(loop_thr=0.0)
    imgs, deps, fpl = view_frames(n, 41)
    gps, poses, enabled = stage_inputs(fpl)
    ep = EpipolarParams(8, 3.0, 0.99)
    pp = Engine.proximity_params(vp, local_radius=1.2)
    st = Engine.decide_stages(n, gps, GPS_RADIUS, ep, pp, poses, enabled)
    ra = Run(a, imgs, deps, op, ns, vp, np.arange(n), dp, st)
    n_pnp = n_ok = 0
    for f in range(n):
        op_f, vp_f = with_k(op, Ks[f]), with_k(vp, Ks[f])
        pp_f = Engine.proximity_params(vp_f, local_radius=1.2)
        st_f = Engine.decide_stages(1, gps[f:f + 1], GPS_RADIUS, ep, pp_f, poses[f:f + 1], enabled[f:f + 1])
        rb = Run(b, imgs[f:f + 1], deps[f:f + 1], op_f, ns, vp_f, [f], dp, st_f)
        assert ra.frame(f) == rb.frame(0), f"frame {f}"
        # the registrations of the frame: its decision's, or the proximity paths' when one of them took the decision's place
        regs = [ra.results()[f]] + [p["result"] for p in Engine.proximity_records(ra.prox)[f]["paths"]]
        n_pnp += any(r["n_matches"] >= vp.min_inliers for r in regs)
        n_ok += any(r["ok"] for r in regs)
    assert n_pnp >= 16 and n_ok >= 1, f"PnP ran for {n_pnp} frames, {n_ok} registrations succeeded"


def oracle_registration(b, imgs, deps, op, f, place, L, vp):
    """the oracle's registration of frame f against stored place `place`, TO = the frame's detected rows lifted with L"""
    w, _ = world(DETECTOR_ORB)
    desc_s, xyz_s, _, _ = map_arrays(DETECTOR_ORB)
    row = list(w.smap.sig_ids).index(place)
    nf = int(w.smap.ni[row])
    kp, desc, xyz = b.orb_detect_describe(imgs[f:f + 1], deps[f:f + 1], op, cap=DET)[0]
    return co.register(desc_s[row][:nf], xyz_s[row][:nf], desc, kp[:, :2], K4, xyz_to=co.lift(xyz, L), L=L, image_size=(vp.image_width, vp.image_height),
                       repeat_once=bool(vp.repeat_once), guess_win_size=vp.guess_win_size)


def test_local_transforms_against_the_oracle():
    n = 24
    a, places = load(DETECTOR_ORB)
    a.clients_create(n)
    Ls = local_transforms(n)
    a.clients_set_cameras(range(n), [camera_model(K4, (W, H), L) for L in Ls])
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4, image_size=(W, H), repeat_once=True)
    imgs, deps, _ = view_frames(n, 43)
    r = Run(a, imgs, deps, op, len(places), vp, np.arange(n), Engine.decide_params(loop_thr=0.0))
    res = r.results()
    checked = 0
    for f in range(n):
        if r.dec[f]["status"] not in (ACCEPTED, VERIFY_REJECTED):
            continue
        o = oracle_registration(a, imgs, deps, op, f, int(r.dec[f]["highest_id"]), Ls[f], vp)
        g = res[f]
        assert (g["ok"], g["n_matches"], g["n_inliers"]) == (o["ok"], len(o["matches"]), len(o["inliers"])), f"frame {f}"
        if o["ok"]:
            checked += 1
            np.testing.assert_allclose(g["rvec"], o["rvec"], atol=1e-4)
            np.testing.assert_allclose(g["tvec"], o["tvec"], atol=1e-4)
            np.testing.assert_allclose(g["transform"], o["transform"], atol=1e-4)
            np.testing.assert_allclose(g["covariance"], o["covariance"], atol=1e-4)
    assert checked >= 8, checked


def norms(run):
    return np.array([np.linalg.norm(r["transform"][:, 3]) if r["ok"] else np.nan for r in run.results()])


def test_distance_checks_read_the_base_frame_transform():
    """RGBD/MaxLoopClosureDistance between the camera-frame and the base-frame norm rejects only with the local transform set; the
    proximity radius test the same way"""
    n = 24
    Ls = local_transforms(n, seed=5)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4)
    imgs, deps, fpl = view_frames(n, 47)

    def run(with_cam, max_dist, pp=None):
        e, places = load(DETECTOR_ORB)
        e.clients_create(n)
        if with_cam:
            e.clients_set_cameras(range(n), [camera_model(K4, (0, 0), L) for L in Ls])
        st = None
        if pp is not None:
            gps, poses, enabled = stage_inputs(fpl)
            st = Engine.decide_stages(n, None, GPS_RADIUS, None, pp, poses, enabled)
        r = Run(e, imgs, deps, op, len(places), vp, np.arange(n), Engine.decide_params(loop_thr=0.0, max_loop_closure_distance=max_dist), st)
        e.close()
        return r

    nb, nc = norms(run(True, 0.0)), norms(run(False, 0.0))
    gap = np.where(np.isfinite(nb) & np.isfinite(nc), nb - nc, -np.inf)
    f = int(np.argmax(gap))
    assert gap[f] > 0.05, gap
    limit = float((nb[f] + nc[f]) / 2)
    assert run(True, limit).dec[f]["status"] == DISTANCE_REJECTED
    assert run(False, limit).dec[f]["status"] == ACCEPTED
    # proximity: a path accepted without the local transform and refused with it, at a filtering radius between the two norms
    def paths(r):
        return {(f, j): (p["accepted"], np.linalg.norm(p["result"]["transform"][:, 3]) if p["result"]["ok"] else np.nan)
                for f, rec in enumerate(Engine.proximity_records(r.prox)) for j, p in enumerate(rec["paths"])}

    pb = paths(run(True, 0.0, Engine.proximity_params(vp, local_radius=1.2, path_filtering_radius=0.0)))
    pc = paths(run(False, 0.0, Engine.proximity_params(vp, local_radius=1.2, path_filtering_radius=0.0)))
    cand = sorted((pb[k][1] - pc[k][1], k) for k in pb if k in pc and np.isfinite(pb[k][1]) and np.isfinite(pc[k][1]) and pb[k][1] > pc[k][1])
    assert cand, "no proximity registration to test"
    flipped = False
    for _, k in cand[::-1][:3]:
        radius = float((pb[k][1] + pc[k][1]) / 2)
        xb = paths(run(True, 0.0, Engine.proximity_params(vp, local_radius=1.2, path_filtering_radius=radius)))
        xc = paths(run(False, 0.0, Engine.proximity_params(vp, local_radius=1.2, path_filtering_radius=radius)))
        if any(xc[q][0] and not xb.get(q, (True,))[0] for q in xc):
            flipped = True
            break
    assert flipped, "the proximity radius test did not read the base-frame transform"


def test_mixed_batch_leaves_clients_without_camera_untouched():
    n = 32
    a, places = load(DETECTOR_ORB)
    b, _ = load(DETECTOR_ORB)
    for e in (a, b):
        e.clients_create(n)
    with_cam = np.arange(0, n, 2)
    Ks, Ls = ks(n, 7), local_transforms(n, 8)
    a.clients_set_cameras(with_cam, [camera_model(Ks[c], (W, H), Ls[c]) for c in with_cam])
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4, image_size=(W, H), repeat_once=True)
    pp = Engine.proximity_params(vp, local_radius=1.2)
    dp = Engine.decide_params(loop_thr=0.0, max_loop_closure_distance=2.0)
    for step in range(2):
        imgs, deps, fpl = view_frames(n, 50 + step)
        gps, poses, enabled = stage_inputs(fpl)
        st = Engine.decide_stages(n, gps, GPS_RADIUS, EpipolarParams(8, 3.0, 0.99), pp, poses, enabled)
        clients = np.random.default_rng(step).permutation(n)
        ra = Run(a, imgs, deps, op, len(places), vp, clients, dp, st)
        rb = Run(b, imgs, deps, op, len(places), vp, clients, dp, st)
        for f in range(n):
            if clients[f] % 2:
                assert ra.frame(f) == rb.frame(f), f"step {step} frame {f}"


def test_a_batch_in_flight_keeps_its_cameras():
    n = 16
    a, places = load(DETECTOR_ORB)
    b, _ = load(DETECTOR_ORB)
    cams = [camera_model(k, (W, H), L) for k, L in zip(ks(n, 9), local_transforms(n, 10))]
    for e in (a, b):
        e.clients_create(n)
        e.clients_set_cameras(range(n), cams)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4, image_size=(W, H), repeat_once=True)
    dp = Engine.decide_params(loop_thr=0.0)
    imgs, deps, _ = view_frames(n, 53)
    ra = Run(a, imgs, deps, op, len(places), vp, np.arange(n), dp, between=lambda: a.clients_set_cameras(range(n), None))
    rb = Run(b, imgs, deps, op, len(places), vp, np.arange(n), dp)
    assert all(ra.frame(f) == rb.frame(f) for f in range(n))
    # the cleared cameras apply from the next call on: it equals a run without cameras
    c, _ = load(DETECTOR_ORB)
    c.clients_create(n)
    Run(c, imgs, deps, op, len(places), vp, np.arange(n), dp)
    imgs2, deps2, _ = view_frames(n, 54)
    r2a = Run(a, imgs2, deps2, op, len(places), vp, np.arange(n), dp)
    r2c = Run(c, imgs2, deps2, op, len(places), vp, np.arange(n), dp)
    assert all(r2a.frame(f) == r2c.frame(f) for f in range(n))


def test_float_engine_per_client_k():
    """a 64-D float engine: lcd_decide_batch_dev + lcd_verify_decided_dev of 32 clients with their own K equal one decision per client
    with that K in lcd_verify_params"""
    import torch

    from bayes_cases import make_graph, n_levels
    from test_gpu_decide import Fleet
    from test_gpu_proximity import F, S
    from test_gpu_verify_f32 import IMG, WIN, near

    dim, B, n_words = 64, 32, 3000
    vocab = synth.make_float_vocabulary(n_words, dim, 1)
    wid = np.arange(1, n_words + 1, dtype=np.int32)
    m = synth.make_map(wid, S, F, seed=2)
    rng = np.random.default_rng(12)
    desc = near(rng, vocab[m.sig_words.reshape(-1) - 1], 0.2).reshape(S, F, dim)
    z = rng.uniform(0.5, 5.0, (S, F)).astype(np.float32)
    xyz = np.stack([rng.uniform(-0.55, 0.55, (S, F)) * z, rng.uniform(-0.4, 0.4, (S, F)) * z, z], -1).astype(np.float32)
    fpl = rng.integers(0, S, B)
    Ks = ks(B, 13)
    q = np.empty((B, F, dim), np.float32)
    uv = np.empty((B, F, 2), np.float32)
    for b_, p in enumerate(fpl):
        perm = rng.permutation(F)
        q[b_] = near(rng, desc[p][perm], 0.4)
        uv[b_] = orc.project_points(xyz[p][perm], Ks[b_], rng.normal(0, 0.05, 3), rng.normal(0, 0.1, 3)) + rng.normal(0, 0.5, (F, 2))

    def engine():
        e = Engine(desc_type=LCD_DESC_F32, desc_dim=dim, max_words=n_words, max_signatures=S + 2, max_queries=F, max_batch=128)
        e.add_words(wid, vocab)
        e.last_word_id = n_words
        e.update()
        e.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
        e.sig_add_batch(m.sig_ids, desc, xyz)
        e.clients_create(B)
        fl = Fleet(B, dp=Engine.decide_params(loop_thr=0.0), eng=e)
        sig = [int(s) for s in m.sig_ids]
        fl.set_map(sig, *make_graph("chain", sig, n_levels(fl.text), np.random.default_rng(5)))
        return e

    a, b = engine(), engine()
    a.clients_set_cameras(range(B), [camera_model(k, IMG) for k in Ks])
    vp = Engine.verify_params(K4, image_size=IMG, repeat_once=True, guess_win_size=WIN)
    dp = Engine.decide_params(loop_thr=0.0)
    _, like = a.localize_batch(q.reshape(-1, dim), B, m.sig_ids, S + 1)
    d_q = torch.from_numpy(np.ascontiguousarray(q).reshape(-1)).cuda()
    d_uv = torch.from_numpy(np.ascontiguousarray(uv).reshape(-1)).cuda()
    d_l = torch.from_numpy(np.ascontiguousarray(like, np.float32)).cuda()
    torch.cuda.synchronize()
    a.decide_batch_dev(d_l.data_ptr(), B, S, np.arange(B), np.zeros(B, np.int32), dp)
    a.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, vp)
    hyp, res = a.process_fetch(B)
    dec = a.decide_fetch(B)
    n_ok = 0
    for f in range(B):
        vp_f = with_k(vp, Ks[f])
        b.decide_batch_dev(d_l[f:f + 1].data_ptr(), 1, S, [f], np.zeros(1, np.int32), dp)
        b.verify_decided_dev(d_q[f * F * dim:].data_ptr(), d_uv[f * F * 2:].data_ptr(), 1, F, vp_f)
        hb, rb = b.process_fetch(1)
        assert dec[f].tobytes() == b.decide_fetch(1)[0].tobytes() and hyp[f] == hb[0], f"frame {f}"
        for k in ("ok", "n_matches", "n_inliers", "iterations_run"):
            assert res[f][k] == rb[0][k], f"frame {f}: {k}"
        for k in ("rvec", "tvec", "transform", "covariance"):
            assert np.array_equal(np.asarray(res[f][k]), np.asarray(rb[0][k])), f"frame {f}: {k}"
        n_ok += res[f]["ok"]
    assert n_ok >= B // 4, n_ok


def test_refusals_change_nothing():
    n = 8
    a, places = load(DETECTOR_ORB)
    b, _ = load(DETECTOR_ORB)
    cams = [camera_model(k, (W, H), L) for k, L in zip(ks(n, 14), local_transforms(n, 15))]
    for e in (a, b):
        e.clients_create(n)
        e.clients_set_cameras(range(n), cams)
    good = camera_model(K4, (W, H))

    def bad(**kw):
        c = camera_model(K4, (W, H))
        for k, v in kw.items():
            if k == "L":
                c.local_transform[:] = [float(x) for x in np.asarray(v, np.float32).reshape(-1)]
            else:
                setattr(c, k, v)
        return c

    skew = np.eye(3, 4, dtype=np.float32)
    skew[0, 1] = 1e-3
    for clients, cl in (([0, n], [good, good]), ([-1], [good]), ([0, 1], [good, bad(fx=float("nan"))]), ([1], [bad(cy=float("inf"))]),
                        ([2], [bad(fx=0.0)]), ([2], [bad(fy=-500.0)]), ([3], [bad(L=np.full((3, 4), np.nan, np.float32))]), ([4], [bad(L=skew)]),
                        ([5], [bad(L=2 * np.eye(3, 4, dtype=np.float32))])):
        with pytest.raises(LcdError) as ex:
            a.clients_set_cameras(clients, cl)
        assert ex.value.code == -1, (clients, ex.value)
    op = Engine.orb_params(K4, n_features=DET)
    vp = Engine.verify_params(K4, image_size=(W, H), repeat_once=True)
    dp = Engine.decide_params(loop_thr=0.0)
    imgs, deps, _ = view_frames(n, 57)
    # a camera whose image size is not the images': refused before any state changes
    a.clients_set_cameras([6], [camera_model(K4, (W // 2, H // 2))])
    with pytest.raises(LcdError) as ex:
        Run(a, imgs, deps, op, len(places), vp, np.arange(n), dp)
    assert ex.value.code == -1
    a.clients_set_cameras([6], [cams[6]])
    ra = Run(a, imgs, deps, op, len(places), vp, np.arange(n), dp)
    rb = Run(b, imgs, deps, op, len(places), vp, np.arange(n), dp)
    assert all(ra.frame(f) == rb.frame(f) for f in range(n))
