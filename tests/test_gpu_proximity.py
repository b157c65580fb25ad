"""Proximity detection by space on the GPU (lcd_clients_set_map_poses / lcd_decide_proximity_dev / lcd_proximity_fetch) against the
restatement of oracle/proximity_py.py fed the GPU's adjusted likelihood.

The scenes: places on parallel lines 3 m apart, 0.5 m apart along a line, with random jitter of the positions and yaws (so path
distances differ by far more than 1e-5 relative and no place sits on the radius or angle boundary, with probability 1), neighbour links
along each line with a break every 9 places.  The first 200 places hold signatures; frame b re-observes place places[b] from a pose a
few centimetres away.  Raw likelihood rows spike on the frame's own place (an accepted hypothesis that proximity registers: same-id
suppression), on a place of the next line (another place registered: different-id suppression) or nowhere."""
import numpy as np
import pytest

from bayes_cases import PATTERNS
from oracle import decide_py as dc
from oracle import proximity_py as px
from oracle.bayes_py import parse_prediction_lc, prediction_columns
from rtabmap_b200 import Engine, LcdError, synth

pytestmark = pytest.mark.gpu

S, F = 200, 200


def yaw_pose(x, y, yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, 0]], np.float32)


def scene(n_places, seed=7):
    rng = np.random.default_rng(seed)
    ids = np.arange(1, n_places + 1, dtype=np.int32)
    k = np.arange(n_places)
    x = (k % 100) * 0.5 + rng.uniform(-0.1, 0.1, n_places)
    y = (k // 100) * 3.0 + rng.uniform(-0.2, 0.2, n_places)
    yaw = rng.uniform(-1.2, 1.2, n_places)
    poses = np.stack([yaw_pose(x[i], y[i], yaw[i]) for i in range(n_places)])
    nbr = {int(i): [] for i in ids}
    for i in range(n_places - 1):
        if (i + 1) % 100 and (i + 1) % 9:
            nbr[int(ids[i])].append(int(ids[i + 1]))
            nbr[int(ids[i + 1])].append(int(ids[i]))
    ptr = np.zeros(n_places + 1, np.int64)
    ptr[1:] = np.cumsum([len(nbr[int(i)]) for i in ids])
    flat = np.array([j for i in ids for j in nbr[int(i)]], np.int32)
    return ids, poses, nbr, ptr, flat


@pytest.fixture(scope="module")
def world():
    vocab = synth.make_binary_vocabulary(49152, 32, 1)
    wid = np.arange(1, 49153, dtype=np.int32)
    m = synth.make_map(wid, S, F, seed=2)
    st = synth.make_signature_store(vocab, wid, m)
    q, uv, places, _ = synth.make_query_frames_geo(st, m, 128)
    return vocab, wid, m, st, q, uv, places


def make_engine(world, n_places, n_clients):
    vocab, wid, m, st, *_ = world
    eng = Engine(max_words=49152, max_signatures=n_places + 2, max_queries=F, max_batch=128)
    eng.add_words(wid, vocab)
    eng.last_word_id = 49152
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.sig_add_batch(m.sig_ids, st.desc, st.xyz)
    eng.clients_create(n_clients)
    return eng


def set_map(eng, ids):
    full = [-1] + [int(i) for i in ids]
    cp, rows, lv = prediction_columns(full, lambda i: {i: 0})
    eng.clients_set_map(full, cp, rows, lv, parse_prediction_lc(PATTERNS["default"]))


def frames(world, ids, poses, B, seed):
    """frame poses next to their places, raw likelihood rows, flags and enabled flags"""
    *_, q, uv, places = world
    rng = np.random.default_rng(seed)
    ns = len(ids)
    fp = np.empty((B, 3, 4), np.float32)
    raw = (rng.random((B, ns)) < 0.02).astype(np.float32) * rng.random((B, ns)).astype(np.float32) * 0.3
    for b in range(B):
        r = int(places[b]) - 1
        fp[b] = poses[r]
        fp[b, 0, 3] += np.float32(rng.uniform(0.03, 0.15))
        fp[b, 1, 3] += np.float32(rng.uniform(0.03, 0.15))
        mode = b % 3
        if mode == 0:
            raw[b, r] = 5.0
        elif mode == 1 and r + 100 < ns:
            raw[b, r + 100] = 5.0
    flags = np.zeros(B, np.int32)
    flags[1::17] = dc.FRAME_HOLD
    flags[2::19] = dc.FRAME_SKIP
    enabled = np.ones(B, np.int32)
    enabled[5::23] = 0
    return fp, raw, flags, enabled


def run(eng, world, ids, poses, B, seed, order=None, pp_kw=None, verify=True, frame_poses=None):
    import torch

    *_, q, uv, places = world
    fp, raw, flags, enabled = frames(world, ids, poses, B, seed)
    if frame_poses is not None:
        fp = np.ascontiguousarray(frame_poses, np.float32)
    order = np.arange(B) if order is None else order
    ns = len(ids)
    d_like = torch.from_numpy(raw[order].reshape(-1)).cuda()
    d_q = torch.from_numpy(q[: B * F].reshape(B, F, -1)[order].reshape(-1)).cuda()
    d_uv = torch.from_numpy(uv[: B * F].reshape(B, F, 2)[order].reshape(-1)).cuda()
    torch.cuda.synchronize()
    dp = Engine.decide_params()
    eng.decide_batch_dev(d_like.data_ptr(), B, ns, order, flags[order], dp)
    dec0 = eng.decide_fetch(B)
    vp = Engine.verify_params(synth.CAMERA_K4)
    pp = Engine.proximity_params(vp, **(pp_kw or {}))
    eng.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, fp[order], enabled[order], pp)
    rec = eng.proximity_fetch(B)
    dec1 = eng.decide_fetch(B)
    hyp = res = None
    if verify:
        eng.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, vp)
        hyp, res = eng.process_fetch(B)
    dec2 = eng.decide_fetch(B)
    adj = eng.adjust_likelihood(raw[order])
    return dict(order=order, fp=fp[order], flags=flags[order], enabled=enabled[order], dec0=dec0, dec1=dec1, dec2=dec2, rec=rec, hyp=hyp,
                res=res, adj=adj, pp=pp_kw or {})


def check(world, ids, poses, nbr, out, check_verify=True, stats=None):
    vocab, wid, m, st, q, uv, places = world
    pose_of = {int(i): poses[k] for k, i in enumerate(ids)}
    kw = out["pp"]
    statuses = set()
    for b, o in enumerate(out["order"]):
        r = out["rec"][b]
        if not out["enabled"][b]:
            assert r["status"] == 0 and r["n_attempts"] == 0
            assert out["dec1"][b].tobytes() == out["dec0"][b].tobytes()
            continue
        use = not out["flags"][b] & (dc.FRAME_SKIP | dc.FRAME_HOLD)
        like = {int(i): out["adj"][b][k + 1] for k, i in enumerate(ids)} if use else {}
        nearest, paths, attempts = px.detect(out["fp"][b], pose_of, nbr, like, stats=stats, **kw)
        assert r["status"] == 1 and r["n_nearest"] == len(nearest) and r["n_paths"] == len(paths), f"frame {b}"
        assert r["n_attempts"] == len(attempts), f"frame {b}"
        for g, ((kl, kid, kd), cand) in zip(r["paths"], attempts):
            assert (g["id"], g["candidate_id"]) == (kid, cand), f"frame {b}"
            assert g["likelihood"].tobytes() == np.float32(kl).tobytes() and g["distance"].tobytes() == np.float32(kd).tobytes(), f"frame {b}"
        # the registrations: as lcd_verify_batch holds them
        if check_verify:
            fq = q[o * F:(o + 1) * F][None]
            fu = uv[o * F:(o + 1) * F][None]
            for g in r["paths"]:
                h = g["candidate_id"]
                if h > S:
                    assert not g["result"]["ok"] and g["result"]["n_matches"] == 0
                    continue
                v = eng_verify(world, h, fq, fu)
                assert g["result"]["ok"] == v["ok"] and g["result"]["n_inliers"] == len(v["inliers"]), f"frame {b} place {h}"
                assert g["result"]["n_matches"] == len(v["matches"]), f"frame {b} place {h}"
                if v["ok"]:
                    assert np.allclose(g["result"]["transform"], v["transform"], atol=1e-4), f"frame {b} place {h}"
        results = [(g["result"]["ok"], g["result"]["transform"]) for g in r["paths"]]
        d0 = out["dec0"][b]
        acc, types, sup, loop, status, skip = px.apply(nearest, attempts, results, int(d0["loop_id"]), int(d0["status"]),
                                                       kw.get("path_filtering_radius", 1.0), kw.get("max_loop_closure_distance", 0.0))
        assert [g["accepted"] for g in r["paths"]] == acc and [g["link_type"] for g in r["paths"]] == types, f"frame {b}"
        assert r["suppressed_id"] == sup, f"frame {b}"
        d1 = out["dec1"][b]
        assert (int(d1["loop_id"]), int(d1["status"])) == (loop, status), f"frame {b}"
        assert d1["highest_id"] == d0["highest_id"] and d1["highest_value"].tobytes() == d0["highest_value"].tobytes()
        if skip and out["res"] is not None:
            assert out["dec2"][b].tobytes() == d1.tobytes() and not out["res"][b]["ok"] and out["res"][b]["n_matches"] == 0, f"frame {b}"
            assert out["hyp"][b] == loop
        statuses.add(status)
        if sup:
            statuses.add(("suppressed", sup == int(d0["loop_id"])))
    return statuses


_verify_engine = {}


def eng_verify(world, h, fq, fu):
    vocab, wid, m, st, *_ = world
    if "e" not in _verify_engine:
        _verify_engine["e"] = Engine()
    return _verify_engine["e"].verify_batch(st.desc[h - 1][None], st.xyz[h - 1][None], fq, fu, synth.CAMERA_K4)[0]


@pytest.mark.parametrize("n_places,B", [(1000, 1), (1000, 37), (10000, 64), (50000, 128)])
def test_candidates_paths_verification_and_decisions(world, n_places, B):
    ids, poses, nbr, ptr, flat = scene(n_places)
    eng = make_engine(world, n_places, B)
    set_map(eng, ids)
    eng.clients_set_map_poses(ids, poses, ptr, flat)
    out = run(eng, world, ids, poses, B, seed=n_places + B)
    st = check(world, ids, poses, nbr, out, check_verify=B <= 64)
    if B >= 37:
        assert dc.ACCEPTED in st and ("suppressed", True) in st and ("suppressed", False) in st, st


def test_parameters_angle_depth_paths_and_distance_cap(world):
    n_places, B = 1000, 48
    ids, poses, nbr, ptr, flat = scene(n_places, seed=11)
    eng = make_engine(world, n_places, B)
    set_map(eng, ids)
    eng.clients_set_map_poses(ids, poses, ptr, flat)
    for kw in (dict(angle=0.0, max_paths=16, max_graph_depth=0, path_filtering_radius=0.0),
               dict(angle=20.0, max_paths=1, max_graph_depth=3, path_filtering_radius=2.0, max_loop_closure_distance=0.4),
               dict(local_radius=4.0, max_paths=5, max_graph_depth=1)):
        eng.clients_create(B)
        out = run(eng, world, ids, poses, B, seed=3, pp_kw=kw)
        check(world, ids, poses, nbr, out, check_verify=False)


def csr(ids, nbr):
    ptr = np.zeros(len(ids) + 1, np.int64)
    ptr[1:] = np.cumsum([len(nbr[int(i)]) for i in ids])
    return ptr, np.array([j for i in ids for j in nbr[int(i)]], np.int32)


def tangle(n_places, seed):
    """places scattered over a 16 m square with ids unrelated to their positions, each linked to 1-3 random places within 2 m, some
    links one way only: graph searches reach places that link only to higher ids (left for a later path) and starts that the ascending-id
    admission does not admit (their second path is lost)"""
    rng = np.random.default_rng(seed)
    ids = np.arange(1, n_places + 1, dtype=np.int32)
    xy = rng.uniform(0, 16, (n_places, 2))
    poses = np.stack([yaw_pose(xy[i, 0], xy[i, 1], rng.uniform(-1.2, 1.2)) for i in range(n_places)])
    nbr = {int(i): [] for i in ids}
    for i in range(n_places):
        near = np.flatnonzero(np.hypot(*(xy - xy[i]).T) < 2.0)
        near = near[near != i]
        for j in rng.choice(near, size=min(len(near), int(rng.integers(1, 4))), replace=False):
            if int(ids[j]) not in nbr[int(ids[i])]:
                nbr[int(ids[i])].append(int(ids[j]))
            if rng.random() < 0.7 and int(ids[i]) not in nbr[int(ids[j])]:
                nbr[int(ids[j])].append(int(ids[i]))
    return (ids, poses, nbr, *csr(ids, nbr))


def line(n_places, seed):
    """one unbroken chain of 300 places 3 cm apart, the other places 40 m away: paths of more than 64 places"""
    rng = np.random.default_rng(seed)
    ids = np.arange(1, n_places + 1, dtype=np.int32)
    x = np.where(ids <= 300, (ids - 1) * 0.03 + rng.uniform(-0.004, 0.004, n_places), 40.0 + rng.uniform(0, 5, n_places))
    poses = np.stack([yaw_pose(x[i], rng.uniform(-0.05, 0.05), rng.uniform(-0.3, 0.3)) for i in range(n_places)])
    nbr = {int(i): [] for i in ids}
    for i in range(1, n_places):
        nbr[i].append(i + 1)
        nbr[i + 1].append(i)
    return (ids, poses, nbr, *csr(ids, nbr))


def test_admission_quirk_lost_paths_and_long_paths(world):
    """getPaths on topologies where the ascending-id admission rejects places, paths are lost and paths exceed 64 places"""
    B = 32
    rng = np.random.default_rng(21)
    for make, n_places, kws in ((tangle, 800, (dict(), dict(max_graph_depth=0, max_paths=16, angle=0.0, path_filtering_radius=0.0))),
                                (line, 600, (dict(max_graph_depth=0, max_paths=4), dict()))):
        ids, poses, nbr, ptr, flat = make(n_places, seed=n_places)
        eng = make_engine(world, n_places, B)
        set_map(eng, ids)
        eng.clients_set_map_poses(ids, poses, ptr, flat)
        if make is tangle:
            fp = np.stack([yaw_pose(*rng.uniform(2, 14, 2), rng.uniform(-1.2, 1.2)) for _ in range(B)])
        else:
            fp = np.stack([yaw_pose(rng.uniform(0, 9), 0.02, rng.uniform(-0.3, 0.3)) for _ in range(B)])
        for kw in kws:
            eng.clients_create(B)
            stats = {}
            out = run(eng, world, ids, poses, B, seed=4, pp_kw=kw, frame_poses=fp)
            check(world, ids, poses, nbr, out, stats=stats)
            if make is tangle:
                assert stats["rejected"] > 0 and stats["lost"] > 0, stats
            else:
                assert stats["longest"] > 64, stats


def test_same_bits_at_any_batch_position(world):
    n_places, B = 2000, 40
    ids, poses, nbr, ptr, flat = scene(n_places, seed=5)
    eng = make_engine(world, n_places, B)
    set_map(eng, ids)
    eng.clients_set_map_poses(ids, poses, ptr, flat)
    a = run(eng, world, ids, poses, B, seed=9, verify=False)
    eng.clients_create(B)
    order = np.random.default_rng(1).permutation(B)
    b = run(eng, world, ids, poses, B, seed=9, order=order, verify=False)
    for i, o in enumerate(order):
        assert flat_rec(a["rec"][o]) == flat_rec(b["rec"][i]), f"frame {o}"
        assert a["dec1"][o].tobytes() == b["dec1"][i].tobytes()


def flat_rec(r):
    paths = [(np.float32(g["likelihood"]).tobytes(), g["id"], np.float32(g["distance"]).tobytes(), g["candidate_id"], g["accepted"],
              g["link_type"], g["result"]["ok"], g["result"]["n_matches"], g["result"]["n_inliers"], g["result"]["transform"].tobytes())
             for g in r["paths"]]
    return (r["status"], r["n_nearest"], r["n_paths"], r["n_attempts"], r["suppressed_id"], paths)


def test_stale_poses_and_errors(world):
    import torch

    n_places, B = 1100, 2
    ids, poses, nbr, ptr, flat = scene(n_places)
    eng = make_engine(world, n_places, B)
    vp = Engine.verify_params(synth.CAMERA_K4)
    pp = Engine.proximity_params(vp)

    def code(f):
        with pytest.raises(LcdError) as ex:
            f()
        return ex.value.code

    assert code(lambda: eng.clients_set_map_poses(ids, poses, ptr, flat)) == -4                 # no map
    set_map(eng, ids)
    assert code(lambda: eng.clients_set_map_poses(ids[1:], poses[1:], ptr[1:] - ptr[1], flat[ptr[1]:])) == -1
    bad_ids = ids.copy()
    bad_ids[5] = 99999
    assert code(lambda: eng.clients_set_map_poses(bad_ids, poses, ptr, flat)) == -1
    bad = poses.copy()
    bad[3, 1, 3] = np.nan
    assert code(lambda: eng.clients_set_map_poses(ids, bad, ptr, flat)) == -1
    d_like = torch.zeros(B * n_places, dtype=torch.float32, device="cuda")
    d_q = torch.zeros(B * F * 32, dtype=torch.uint8, device="cuda")
    d_uv = torch.zeros(B * F * 2, dtype=torch.float32, device="cuda")
    en = [1] * B
    prox = lambda p=pp, n=B: eng.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), n, F, poses[:n], [1] * n, p)
    assert code(prox) == -4                                                                     # no decision
    eng.decide_batch_dev(d_like.data_ptr(), B, n_places, [0, 1], [0, 0], Engine.decide_params())
    assert code(prox) == -4                                                                     # no poses
    eng.clients_set_map_poses(ids, poses, ptr, flat)
    assert code(lambda: prox(n=1)) == -1                                                        # not the decision's frame count
    assert code(lambda: prox(Engine.proximity_params(vp, max_paths=0))) == -3
    assert code(lambda: prox(Engine.proximity_params(vp, max_paths=17))) == -3
    assert code(lambda: prox(Engine.proximity_params(vp, local_radius=0.0))) == -1
    assert code(lambda: prox(Engine.proximity_params(vp, max_graph_depth=-1))) == -1
    assert code(lambda: eng.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, np.full((B, 3, 4), np.inf), en, pp)) == -1
    prox()
    assert code(prox) == -4                                                                     # already ran on this decision
    assert code(lambda: prox(Engine.proximity_params(vp, max_paths=-1))) == -3                  # unlimited: not supported
    assert len(eng.proximity_fetch(B)) == B
    # a new map makes the poses stale
    set_map(eng, ids)
    eng.decide_batch_dev(d_like.data_ptr(), B, n_places, [0, 1], [0, 0], Engine.decide_params())
    assert code(prox) == -4
    eng.clients_set_map_poses(ids, poses, ptr, flat)
    prox()
    assert [r["status"] for r in eng.proximity_fetch(B)] == [1, 1]
    # a decision that was already verified: the proximity step comes before the verification
    eng.decide_batch_dev(d_like.data_ptr(), B, n_places, [0, 1], [0, 0], Engine.decide_params())
    eng.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, vp)
    assert code(prox) == -4
    # 1100 places inside the radius, more than a frame can segment: a capacity status, the decision untouched
    dense = poses.copy()
    dense[:, 0, 3] = np.linspace(0, 1, n_places, dtype=np.float32)
    dense[:, 1, 3] = 0
    eng.clients_set_map_poses(ids, dense, ptr, flat)
    eng.decide_batch_dev(d_like.data_ptr(), B, n_places, [0, 1], [0, 0], Engine.decide_params())
    dec0 = eng.decide_fetch(B)
    eng.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, dense[:B], en, pp)
    assert code(lambda: eng.proximity_fetch(B + 1)) == -1
    r = eng.proximity_fetch(B)
    assert [(x["status"], x["n_nearest"], x["n_attempts"]) for x in r] == [(2, n_places, 0)] * B
    assert eng.decide_fetch(B).tobytes() == dec0.tobytes()
