"""A localisation map opened from an RTAB-Map database (dbio.open_localization_map) must leave an engine in the state a caller reaches by
setting every table by hand: a synthetic world with poses, links, GPS and global descriptors is written into a database, opened on one
engine and set up directly from the in-memory arrays on another, and every decision call must answer bit for bit the same.  The
decisions on the loaded tables also follow the restated Bayes filter and Rtabmap::process (oracle/), and a refused database leaves the
engine it was opened on as it was."""
import numpy as np
import pytest

from oracle import decide_py as dc
from oracle import feature2d_py as f2d
from oracle.bayes_py import BayesFilterOracle, graph_tables, prediction_columns
from rtabmap_b200 import Engine, dbio, graph, synth
from test_dbio_map import make_map_db, relative, yaw_pose

pytestmark = pytest.mark.gpu

K4 = (262.5, 262.5, 160.0, 120.0)
B = 24


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def world(tmp_path_factory):
    p = f2d.OrbParams(n_features=600)
    w = synth.make_place_world(lambda img, dep: f2d.detect_describe(img, dep, K4, p), n_places=5, n_words=2800, n_signatures=120, feats=600,
                               height=240, width=320, seed=9)
    rng = np.random.default_rng(3)
    S, F = w.smap.sig_words.shape
    ni = w.smap.ni
    # each signature's rows in the order the database returns them (ORDER BY word_id, ties in written order)
    order = np.stack([np.argsort(np.where(np.arange(F) < ni[s], w.smap.sig_words[s], np.iinfo(np.int32).max), kind="stable") for s in range(S)])
    words = np.take_along_axis(w.smap.sig_words, order, 1)
    desc = np.take_along_axis(w.store.desc, order[:, :, None], 1)
    xyz = np.take_along_axis(w.store.xyz, order[:, :, None], 1)
    fin = np.isfinite(xyz).all(2)
    uv = np.where(fin[..., None], np.stack([K4[0] * xyz[..., 0] / xyz[..., 2] + K4[2], K4[1] * xyz[..., 1] / xyz[..., 2] + K4[3]], 2),
                  rng.uniform(0, 240, (S, F, 2))).astype(np.float32)
    ids = [int(s) for s in w.smap.sig_ids]
    poses = {s: yaw_pose(0.4 * s, 0.3 * (s % 7), 0.02 * s) for s in ids}
    pairs = [(s, s + 1) for s in ids[:-1] if s % 40]                     # three sessions' chains
    loops = [(s, s + 25) for s in ids[:-25:9]]                          # loop closures between revisits
    links = []
    for a, b in pairs:
        links += [(a, b, graph.NEIGHBOR, relative(poses[a], poses[b])), (b, a, graph.NEIGHBOR, relative(poses[b], poses[a]))]
    for a, b in loops:
        links += [(a, b, graph.GLOBAL_CLOSURE, relative(poses[a], poses[b])), (b, a, graph.GLOBAL_CLOSURE, relative(poses[b], poses[a]))]
    gps = {s: (1000.0 + s, -73.6 + 2e-5 * s, 45.5 + 1e-5 * (s % 7), 30.0, 3.0, 20.0 * (s % 18)) for s in ids if s % 10 == 3}
    gdesc = np.abs(rng.normal(size=(S, 32))).astype(np.float32)
    feats = [(s, int(words[k, j]), uv[k, j, 0], uv[k, j, 1], None if not fin[k, j] else xyz[k, j], desc[k, j].tobytes())
             for k, s in enumerate(ids) for j in range(int(ni[k]))]
    db = str(tmp_path_factory.mktemp("db") / "map.db")
    opt = np.stack([poses[s] for s in ids])
    make_map_db(db, w.word_ids, w.vocab, ids, feats, links, (np.array(ids, np.int32), opt), gps,
                [(s, 1, gdesc[k:k + 1]) for k, s in enumerate(ids)], poses=poses)
    return dict(w=w, db=db, ids=ids, words=words, desc=desc, xyz=xyz, uv=uv, ni=ni, poses=poses, opt=opt, pairs=pairs, loops=loops,
                links=links, gps=gps, gdesc=gdesc)


def new_engine():
    e = Engine(max_words=4096, max_signatures=256, max_queries=600, max_batch=B)
    e.clients_create(B)
    return e


def direct(W):
    """today's calls on the in-memory arrays"""
    w, ids = W["w"], W["ids"]
    e = new_engine()
    e.add_words(w.word_ids, w.vocab)
    e.last_word_id = int(w.word_ids.max())
    e.update()
    e.load_csr(w.smap.word_ids, w.smap.row_ptr, w.smap.sig, w.smap.cnt)
    e.set_ni(w.smap.sig_ids, w.smap.ni)
    e.sig_add_batch(ids, W["desc"], W["xyz"], W["ni"])
    e.sig_words_add_batch(ids, W["words"], W["uv"], W["ni"])
    lc = graph.DEFAULT_PREDICTION_LC
    tables = graph_tables(ids, len(lc) - 2, W["pairs"], W["loops"])
    full = [-1] + ids
    cp, rows, lv = prediction_columns(full, tables.__getitem__)
    e.clients_set_map(full, cp, rows, lv, lc, 0.9)
    nbr = {s: sorted([b for a, b in W["pairs"] if a == s] + [a for a, b in W["pairs"] if b == s]) for s in ids}
    ptr = np.concatenate([[0], np.cumsum([len(nbr[s]) for s in ids])]).astype(np.int64)
    e.clients_set_map_poses(ids, W["opt"], ptr, np.array([b for s in ids for b in nbr[s]], np.int32))
    g6 = np.array([W["gps"].get(s, (0.0,) * 6) for s in ids], np.float64)
    ln = dbio.Links(np.array([l[0] for l in W["links"]], np.int32), np.array([l[1] for l in W["links"]], np.int32),
                    np.array([l[2] for l in W["links"]], np.int32), np.stack([l[3] for l in W["links"]]))
    order = np.lexsort((ln.to_id, ln.from_id))
    ln = dbio.Links(ln.from_id[order], ln.to_id[order], ln.type[order], ln.transform[order])
    gps, off = graph.gps_of_places(ids, g6, np.stack([W["poses"][s] for s in ids]), ln)
    e.clients_set_map_gps(ids, gps[:, :5], off)
    e.gdesc_add(ids, W["gdesc"])
    return e, tables


def same_results(a, b, where):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        for key in x:
            assert np.array_equal(np.asarray(x[key]), np.asarray(y[key])), f"{where} frame {k}: {key}"


def test_loaded_engine_answers_like_the_hand_set_one(world):
    import torch

    W = world
    ids = W["ids"]
    ns = len(ids)
    loaded = new_engine()
    res = dbio.open_localization_map(loaded, W["db"])
    assert list(res.places) == ids and res.poses_set and res.gps_set and res.n_global_descriptors == ns and res.skipped == {}
    assert res.n_gps_offsets > 0 and loaded.sig_count() == ns and loaded.sig_words_count == ns and loaded.gdesc_count() == ns
    hand, tables = direct(W)
    st = synth.SynthStore(W["desc"], W["xyz"])
    q, uv, places, _ = synth.make_query_frames_geo(st, W["w"].smap, B, seed=5, K4=K4)
    F = len(q) // B
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_uv = torch.from_numpy(uv.reshape(-1)).cuda()
    d_s = torch.tensor(ids, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(6)
    clients = rng.permutation(B)
    flags = np.zeros(B, np.int32)
    flags[::7] = dc.FRAME_AGGRESSIVE
    vp = Engine.verify_params(K4)
    dp = Engine.decide_params()
    fpose = np.stack([W["poses"][int(p)] for p in places]).astype(np.float32)
    fpose[:, :2, 3] += 0.05
    pp = Engine.proximity_params(vp, local_radius=2.0)
    frame_gps = np.array([(1.0, -73.6 + 2e-5 * int(p), 45.5 + 1e-5 * (int(p) % 7), 30.0, 2.0) for p in places])
    frame_gps[::5, 0] = 0.0
    out = []
    for e in (loaded, hand):
        o = {}
        d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
        d_l = torch.zeros(B * ns, dtype=torch.float32, device="cuda")
        d_p = torch.zeros(B * (ns + 1), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        e.process_decide_batch_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, ns, ns + 1, vp, clients, flags, dp, d_w.data_ptr(), d_l.data_ptr(),
                                   d_p.data_ptr())
        o["dec"] = e.decide_fetch(B)
        o["decide"] = o["dec"].tobytes()
        o["hyp"], o["res"] = e.process_fetch(B)
        o["words"], o["like"], o["post"] = d_w.cpu().numpy(), d_l.cpu().numpy().reshape(B, ns), d_p.cpu().numpy().reshape(B, ns + 1)
        # the decomposed path on the same likelihood: decide, epipolar check, proximity, then verification
        d_p2 = torch.zeros(B * (ns + 1), dtype=torch.float32, device="cuda")
        e.decide_batch_dev(d_l.data_ptr(), B, ns, clients, flags, dp, d_p2.data_ptr())
        o["decide2"] = e.decide_fetch(B).tobytes()
        o["post2"] = d_p2.cpu().numpy()
        d_n = torch.full((B,), F, dtype=torch.int32, device="cuda")
        e.decide_epipolar_dev(d_w.data_ptr(), d_uv.data_ptr(), d_n.data_ptr(), B, F)
        o["epi"] = e.epipolar_fetch(B)
        o["decide_epi"] = e.decide_fetch(B).tobytes()
        e.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, fpose, np.ones(B, np.int32), pp)
        o["prox"] = e.proximity_fetch(B)
        o["decide_prox"] = e.decide_fetch(B).tobytes()
        e.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, vp)
        o["hyp2"], o["res2"] = e.process_fetch(B)
        d_c = torch.zeros(B * ns, dtype=torch.uint8, device="cuda")
        e.decide_gps_batch_dev(d_l.data_ptr(), B, ns, clients, flags, frame_gps, 50.0, dp, d_p.data_ptr(), d_c.data_ptr())
        o["decide_gps"] = e.decide_fetch(B).tobytes()
        o["post_gps"], o["compared"] = d_p.cpu().numpy(), d_c.cpu().numpy()
        d_g = torch.from_numpy(W["gdesc"][[int(p) - 1 for p in places]] + np.float32(0.01)).cuda()
        d_ls = torch.zeros(B * ns, dtype=torch.float32, device="cuda")
        e.localize_similarity_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), ns, d_g.data_ptr(), 0, d_ls.data_ptr())
        e.synchronize()
        o["sim"] = d_ls.cpu().numpy()
        out.append(o)
    a, b = out
    for key in ("decide", "decide2", "decide_epi", "decide_prox", "decide_gps"):
        assert a[key] == b[key], key
    for key in ("hyp", "hyp2", "words", "compared"):
        assert np.array_equal(a[key], b[key]), key
    for key in ("like", "post", "post2", "post_gps", "sim"):
        assert np.array_equal(bits(a[key]), bits(b[key])), key
    same_results(a["res"], b["res"], "process_decide")
    same_results(a["res2"], b["res2"], "verify_decided")
    for x, y in zip(a["epi"], b["epi"]):
        assert all(np.array_equal(np.asarray(x[k]), np.asarray(y[k])) for k in x)
    for x, y in zip(a["prox"], b["prox"]):
        assert {k: v for k, v in x.items() if k != "paths"} == {k: v for k, v in y.items() if k != "paths"}
        assert len(x["paths"]) == len(y["paths"])
        for p, r in zip(x["paths"], y["paths"]):
            assert {k: v for k, v in p.items() if k != "result"} == {k: v for k, v in r.items() if k != "result"}
            same_results([p["result"]], [r["result"]], "proximity")
    assert (a["compared"] == 0).any(), "the GPS filter compared every place"
    assert any(x["n_pairs"] for x in a["epi"]) and any(r["status"] == 1 and r["n_attempts"] for r in a["prox"])
    # the decisions on the loaded tables, end to end: the restated filter and Rtabmap::process
    dec = a["dec"]
    adj = loaded.adjust_likelihood(a["like"])
    nb = graph.bayes_neighbors(ids, dbio.read_links(W["db"]), len(graph.DEFAULT_PREDICTION_LC) - 1)
    assert nb == tables
    full = [-1] + ids
    statuses = set()
    for k in range(B):
        bf = BayesFilterOracle(graph.DEFAULT_PREDICTION_LC, 0.9)
        want_post = bf.compute_posterior_sparse(full, adj[k], nb.__getitem__)
        assert np.allclose(a["post"][k], want_post, rtol=1e-4, atol=1e-9) and np.argmax(a["post"][k]) == np.argmax(want_post), f"frame {k}"
        want = dc.DecideClient().decide(full, a["post"][k], int(flags[k]))
        got = (int(dec[k]["highest_id"]), int(dec[k]["loop_id"]), int(dec[k]["status"]))
        assert got[0] == want[0], f"frame {k}"
        if want[3] == dc.ACCEPTED:
            assert got[2] in (dc.ACCEPTED, dc.VERIFY_REJECTED, dc.DISTANCE_REJECTED) and got[1] in (want[2], 0), f"frame {k}"
        else:
            assert got[1:] == (want[2], want[3]), f"frame {k}"
        statuses.add(got[2])
    assert dc.ACCEPTED in statuses


def test_a_refused_database_leaves_the_engine_as_it_was(world, tmp_path):
    import torch

    W = world
    eng, _ = direct(W)
    st = synth.SynthStore(W["desc"], W["xyz"])
    q, uv, places, _ = synth.make_query_frames_geo(st, W["w"].smap, 4, seed=8, K4=K4)
    F = len(q) // 4

    def localise():
        d_q = torch.from_numpy(q.reshape(-1)).cuda()
        d_uv = torch.from_numpy(uv.reshape(-1)).cuda()
        d_l = torch.zeros(4 * len(W["ids"]), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        eng.process_decide_batch_dev(d_q.data_ptr(), d_uv.data_ptr(), 4, F, len(W["ids"]), len(W["ids"]) + 1, Engine.verify_params(K4),
                                     [0, 1, 2, 3], [0, 0, 0, 0], Engine.decide_params(), 0, d_l.data_ptr())
        return bits(d_l.cpu().numpy()), eng.process_fetch(4)[0]

    eng.clients_reset(list(range(B)))
    before = localise()
    w = W["w"]
    feats = [(1, int(w.word_ids[0]), 1.0, 1.0, None, w.vocab[0].tobytes())] * 4100 + [(2, int(w.word_ids[1]), 1.0, 1.0, None, w.vocab[1].tobytes())]
    for name, kw in (("capacity", {}), ("intermediate", dict(weights={2: -1}))):
        db = str(tmp_path / f"{name}.db")
        make_map_db(db, w.word_ids[:50], w.vocab[:50], [1, 2], feats, **kw)
        with pytest.raises(dbio.DbFormatError) as ex:
            dbio.open_localization_map(eng, db)
        if name == "capacity":
            assert "at most 4096" in str(ex.value)
    eng.clients_reset(list(range(B)))
    after = localise()
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    assert eng.sig_count() == len(W["ids"]) and eng.gdesc_count() == len(W["ids"])
