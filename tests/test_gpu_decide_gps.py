"""The GPS filter of the place list (Rtabmap/LoopGPS) in the batched decision of localisation clients (lcd_clients_set_map_gps /
lcd_decide_gps_batch_dev).

Compared places: exactly the restated gate (oracle/gps_py.py, pinned to the reference's GeodeticCoords.cpp by tests/test_oracle_gps.py).
Posterior: per frame over its compared places, against the sparse restatement (oracle/bayes_py.py) and, for two clients, the reference's
compiled BayesFilter.cpp, with the bars of tests/test_gpu_decide.py; 0 at every place the frame did not compare.  Decisions: exactly
the restated Rtabmap::process fed the GPU's posterior over the compared places."""
import numpy as np
import pytest

import gps_cases as gc
from bayes_cases import PATTERNS, make_graph, n_levels
from oracle import decide_py as dc
from oracle import gps_py as gp
from rtabmap_b200 import Engine, LcdError, synth
from test_gpu_decide import ACTIVE_MASK, UNTOUCHED, Fleet, bits, check_float_sum, check_posterior, random_flags, raw_rows, sparse_step

pytestmark = pytest.mark.gpu


def code(f):
    with pytest.raises(LcdError) as ex:
        f()
    return ex.value.code


class GpsFleet(Fleet):
    def set_map_gps(self, gps, off):
        self.gmap = gp.GpsMap(gps, off)
        self.eng.clients_set_map_gps(self.ids[1:], gps, off)

    def run_gps(self, clients, raw, flags, frame_gps, radius):
        import torch

        B, ns = raw.shape
        d_like = torch.from_numpy(np.ascontiguousarray(raw).reshape(-1)).cuda()
        d_post = torch.full((B * (ns + 1),), UNTOUCHED, dtype=torch.float32, device="cuda")
        d_cmp = torch.full((B * ns,), 7, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        self.eng.decide_gps_batch_dev(d_like.data_ptr(), B, ns, clients, flags, frame_gps, radius, self.dp, d_post.data_ptr(), d_cmp.data_ptr())
        dec = self.eng.decide_fetch(B)
        return dec, d_post.cpu().numpy().reshape(B, ns + 1), d_cmp.cpu().numpy().reshape(B, ns).astype(bool)

    def step_gps(self, clients, raw, flags, frame_gps, radius, where="", restate=None):
        """the GPU call, then every frame against the restatement; restate: the frames whose posterior is checked (default all)"""
        clients = [int(c) for c in clients]
        dec, post, cmp = self.run_gps(clients, raw, flags, frame_gps, radius)
        ids_all = np.array(self.ids)
        for b, c in enumerate(clients):
            w = f"{where} frame {b} client {c}"
            active = not flags[b] & ACTIVE_MASK
            want_cmp = gp.gate(self.gmap, frame_gps[b], radius) if active else np.zeros(len(ids_all) - 1, bool)
            assert np.array_equal(cmp[b], want_cmp), f"{w}: compared places differ ({int(cmp[b].sum())} vs {int(want_cmp.sum())})"
            sel = np.concatenate([[True], want_cmp])
            ids = [int(i) for i in ids_all[sel]]
            if active:
                assert (post[b][~sel] == 0).all(), w + ": a place that was not compared has a posterior"
                adj = gp.GpsClient.adjusted(raw[b], want_cmp, self.dp.virtual_place_ratio)
                if restate is None or b in restate:
                    cols = self.cols if sel.all() else gp.sparse_columns(self.sparse[c], ids, self.tables.__getitem__, self.stm)
                    o, od = sparse_step(self.sparse[c], ids, adj, cols)
                    check_posterior(post[b][sel], od, w + " vs sparse restatement (double sum)")
                    check_float_sum(post[b][sel], o, w + " vs sparse restatement")
                else:   # keep the restatement's state: the GPU posterior, re-keyed
                    self.sparse[c].posterior = {i: np.float32(v) for i, v in zip(ids, post[b][sel])}
                if c in self.refs:
                    self.refs[c].set_graph(self.tables, self.stm)
                    r = self.refs[c].compute_posterior(ids, adj)
                    check_float_sum(post[b][sel], r, w + " vs reference")
            else:
                assert (post[b] == np.float32(UNTOUCHED)).all(), w + ": a skipped / held frame's row was written"
            last = float(self.dec[c].highest[1])
            want = self.dec[c].decide(ids, post[b][sel] if active else None, int(flags[b]))
            got = (int(dec[b]["highest_id"]), np.float32(dec[b]["highest_value"]), int(dec[b]["loop_id"]), int(dec[b]["status"]))
            assert got[0] == want[0] and bits(got[1]) == bits(want[1]) and got[2:] == want[2:], f"{w}: {got} != {want}"
            self.statuses.add(got[3])
            if c in self.refs and active:
                rd = self.dec_ref[c].decide(ids, r, int(flags[b]))
                thr = (self.dp.loop_thr, self.dp.aggressive_loop_thr, self.dp.loop_ratio * last)
                top = np.sort(r[1:].astype(np.float64))[-2:]
                tie = len(top) == 2 and top[1] - top[0] <= 1e-4 * top[1]
                if not tie and all(abs(float(want[1]) - t) > 1e-3 for t in thr):
                    assert rd[0] == want[0] and rd[2:] == want[2:], f"{w}: decision on the reference posterior {rd} != {want}"
            if c in self.refs:
                self.dec_ref[c].highest = self.dec[c].highest
        return dec, post, cmp


def frames_gps(rng, pos, B, share_fix=0.8):
    out = []
    for _ in range(B):
        if rng.random() < share_fix:
            out.append(gc.frame_gps_near(pos[int(rng.integers(len(pos)))], rng))
        else:
            out.append((0.0, 0.0, 0.0, 0.0, 0.0))
    return np.array(out, np.float64)


def radius_for_share(gmap, fr, share):
    """a radius that keeps about `share` of the places around fix fr"""
    _, lon, lat, alt, _ = fr
    e = gp.enu(gmap.geo, gp.geocentric(lat, lon, alt), lat, lon)
    d = np.sqrt((e ** 2).sum(1))
    return float(np.quantile(d, share)) if share < 1 else float(d.max() * 2 + 100)


@pytest.mark.parametrize("share", [0.01, 0.3, 1.0])
def test_128_clients_10000_places(share):
    """128 clients against 10 000 places, two steps, radii keeping about 1 %, 30 % and 100 % of the places; two clients also against
    the reference's BayesFilter.cpp.  Every frame's compared places and decision are checked; 24 frames' posteriors per step against
    the sparse restatement."""
    rng = np.random.default_rng(int(share * 1000) + 3)
    fl = GpsFleet(128, "trunc5", ref_clients=(5, 77), dp=Engine.decide_params(loop_thr=0.11, loop_ratio=0.3))
    places = list(range(1, 10001))
    fl.set_map(places, *make_graph("chain", places, n_levels(fl.text), rng))
    gps, off, pos = gc.trajectory_gps(10000, rng, spacing=4.0, no_fix=0.02, offsets=0.1)
    fl.set_map_gps(gps, off)
    radius = radius_for_share(fl.gmap, gc.gps_row(*pos[5000]), share)
    for t in range(2):
        order = rng.permutation(128)
        fg = frames_gps(rng, pos, 128)
        restate = set(int(b) for b in rng.choice(128, 24, replace=False)) | {int(np.nonzero(order == 5)[0][0]), int(np.nonzero(order == 77)[0][0])}
        flags = random_flags(rng, 128)
        _, _, cmp = fl.step_gps(order, raw_rows(rng, 128, 10000), flags, fg, radius, f"share {share} step {t}", restate)
    kept = cmp[(fg[:, 0] > 0) & ((flags & ACTIVE_MASK) == 0)][:, fl.gmap.fix].mean()   # places without a fix are always compared
    assert (share == 1.0 and kept == 1.0) or (0.2 * share <= kept <= 3 * share), kept


def test_mixed_batch_is_bit_identical_to_the_ungated_call_for_frames_without_a_fix_and_for_a_radius_covering_every_place():
    """Two engines with the same clients: one decides with lcd_decide_batch_dev, the other with lcd_decide_gps_batch_dev where a third of
    the frames carry no fix and the others a fix whose radius covers every place.  Decisions, posterior rows and the clients' state (a
    later ungated step on both) are the same bits; then a gating radius changes the gated frames only."""
    rng = np.random.default_rng(17)
    places = list(range(1, 2001))
    text = PATTERNS["trunc5"]
    tables, stm = make_graph("loops", places, n_levels(text), rng)
    gps, off, pos = gc.trajectory_gps(2000, rng, no_fix=0.05, offsets=0.2)
    a, g = GpsFleet(96, "trunc5"), GpsFleet(96, "trunc5")
    for fl in (a, g):
        fl.set_map(places, tables, stm)
    g.set_map_gps(gps, off)
    huge = 1.0e6
    B = 96
    for t in range(3):
        raw = raw_rows(rng, B, 2000)
        flags = random_flags(rng, B)
        fg = np.array([(0.0,) * 5 if b % 3 == 0 else gc.frame_gps_near(pos[int(rng.integers(2000))], rng) for b in range(B)])
        da, pa = a.run(list(range(B)), raw, flags)
        if t < 2:
            dg, pg, cmp = g.run_gps(list(range(B)), raw, flags, fg, huge)
        else:
            dg, pg = g.run(list(range(B)), raw, flags)
        assert np.array_equal(bits(pa), bits(pg)), f"step {t}: posterior bits differ"
        assert da.tobytes() == dg.tobytes(), f"step {t}: decisions differ"
    # a gating radius changes the gated frames only
    raw = raw_rows(rng, B, 2000)
    flags = np.zeros(B, np.int32)
    fg = np.array([(0.0,) * 5 if b % 2 else gc.frame_gps_near(pos[int(rng.integers(2000))], rng) for b in range(B)])
    da, pa = a.run(list(range(B)), raw, flags)
    dg, pg, cmp = g.run_gps(list(range(B)), raw, flags, fg, 30.0)
    odd = np.arange(B) % 2 == 1
    assert np.array_equal(bits(pa[odd]), bits(pg[odd])) and da[odd].tobytes() == dg[odd].tobytes()
    assert not cmp[~odd].all(axis=1).any(), "the gating radius kept every place"


def test_a_gated_client_gets_the_same_bits_alone_anywhere_in_a_batch():
    rng = np.random.default_rng(8)
    places = list(range(1, 1501))
    tables, stm = make_graph("loops", places, n_levels(PATTERNS["default"]), rng)
    gps, off, pos = gc.trajectory_gps(1500, rng, no_fix=0.05, offsets=0.2)
    steps = [(raw_rows(rng, 128, 1500), random_flags(rng, 128), frames_gps(rng, pos, 128)) for _ in range(3)]
    track_fix = [gc.frame_gps_near(pos[k], rng) for k in (100, 700, 701)]
    runs = []
    for B, pos_b in [(1, 0), (128, 0), (128, 77), (33, 32)]:
        fl = GpsFleet(128)
        fl.set_map(places, tables, stm)
        fl.set_map_gps(gps, off)
        out = []
        for t, (raw, flags, fg) in enumerate(steps):
            others = [c for c in np.random.default_rng(100 * t + pos_b).permutation(128) if c != 9][:B - 1]
            clients = others[:pos_b] + [9] + others[pos_b:]
            rows = raw[:B].copy()
            rows[pos_b] = raw[0]
            fr = flags[:B].copy()
            fr[pos_b] = 0
            g = fg[:B].copy()
            g[pos_b] = track_fix[t]
            dec, post, cmp = fl.run_gps(clients, rows, fr, g, 40.0)
            out.append((bits(post[pos_b]).copy(), dec[pos_b].tobytes(), cmp[pos_b].copy()))
        runs.append(out)
    for r in runs[1:]:
        for t in range(3):
            assert np.array_equal(r[t][0], runs[0][t][0]) and r[t][1] == runs[0][t][1] and np.array_equal(r[t][2], runs[0][t][2]), f"step {t}"


def test_single_hypothesis_and_only_the_virtual_place():
    """A fix far from every place keeps only the virtual place (and the places without a fix); a fix on a place with a small radius keeps
    that one place, and a threshold > 0 rejects it as the single hypothesis."""
    rng = np.random.default_rng(4)
    places = list(range(1, 201))
    fl = GpsFleet(4, dp=Engine.decide_params(loop_thr=0.01))
    fl.set_map(places, *make_graph("loops", places, n_levels(fl.text), rng))
    gps, off, pos = gc.trajectory_gps(200, rng, spacing=6.0)
    fl.set_map_gps(gps, off)
    far = gc.gps_row(pos[0][0] + 9000.0, pos[0][1], error=1.0)
    for t in range(3):
        fg = np.array([far, tuple(gps[50, :4]) + (5.0,), tuple(gps[120, :4]) + (5.0,), (0.0,) * 5])
        _, _, cmp = fl.step_gps([0, 1, 2, 3], raw_rows(rng, 4, 200), np.zeros(4, np.int32), fg, 1.0, f"step {t}")
        assert cmp[0].sum() == 0 and cmp[1].sum() == 1 and cmp[2].sum() == 1 and cmp[3].all()
    assert dc.SINGLE_HYPOTHESIS in fl.statuses


def test_set_map_drops_the_gps_table_and_errors_leave_the_state_in_place():
    import torch

    rng = np.random.default_rng(6)
    places = list(range(1, 101))
    tables, stm = make_graph("loops", places, n_levels(PATTERNS["default"]), rng)
    gps, off, pos = gc.trajectory_gps(100, rng)
    twins = [GpsFleet(3), GpsFleet(3)]
    for fl in twins:
        fl.set_map(places, tables, stm)
    e = twins[0].eng
    raw = raw_rows(rng, 3, 100)
    d = torch.from_numpy(raw.reshape(-1)).cuda()
    dp = Engine.decide_params()
    fix = np.array([gc.frame_gps_near(pos[10], rng)] * 3)
    nofix = np.zeros((3, 5))
    assert code(lambda: e.decide_gps_batch_dev(d.data_ptr(), 3, 100, [0, 1, 2], [0, 0, 0], fix, 10.0, dp)) == -4   # no GPS table yet
    for fl in twins:
        fl.set_map_gps(gps, off)
        fl.run_gps([0, 1, 2], raw, np.zeros(3, np.int32), fix, 25.0)
    before = e.decide_fetch(3).tobytes()
    bad_gps = gps.copy()
    bad_gps[4, 2] = np.nan
    ids = np.array(places, np.int32)
    assert code(lambda: e.clients_set_map_gps(ids, bad_gps, off)) == -1
    assert code(lambda: e.clients_set_map_gps(ids[::-1], gps, off)) == -1
    assert code(lambda: e.clients_set_map_gps(ids[:-1], gps[:-1], off[:-1])) == -1
    bad_off = off.copy()
    bad_off[3, 1] = np.inf
    assert code(lambda: e.clients_set_map_gps(ids, gps, bad_off)) == -1
    for radius in (-1.0, float("nan"), float("inf")):
        assert code(lambda: e.decide_gps_batch_dev(d.data_ptr(), 3, 100, [0, 1, 2], [0, 0, 0], fix, radius, dp)) == -1
    bad_fix = fix.copy()
    bad_fix[1, 1] = np.inf
    assert code(lambda: e.decide_gps_batch_dev(d.data_ptr(), 3, 100, [0, 1, 2], [0, 0, 0], bad_fix, 10.0, dp)) == -1
    assert code(lambda: e.decide_gps_batch_dev(d.data_ptr(), 3, 100, [0, 0, 2], [0, 0, 0], fix, 10.0, dp)) == -1
    assert code(lambda: e.decide_gps_batch_dev(d.data_ptr(), 3, 99, [0, 1, 2], [0, 0, 0], fix, 10.0, dp)) == -1
    assert e.decide_fetch(3).tobytes() == before
    # the failed calls changed nothing: both engines go on with the same bits
    step = (raw_rows(rng, 3, 100), np.zeros(3, np.int32), np.array([gc.frame_gps_near(pos[40], rng)] * 3))
    out = [fl.run_gps([0, 1, 2], *step, 30.0) for fl in twins]
    assert out[0][0].tobytes() == out[1][0].tobytes() and np.array_equal(bits(out[0][1]), bits(out[1][1]))
    # a new map drops the GPS table: fixes are refused, frames without one are decided
    twins[0].set_map(places[:90], *make_graph("loops", places[:90], n_levels(PATTERNS["default"]), rng))
    d2 = torch.from_numpy(raw_rows(rng, 3, 90).reshape(-1)).cuda()
    assert code(lambda: e.decide_gps_batch_dev(d2.data_ptr(), 3, 90, [0, 1, 2], [0, 0, 0], fix, 10.0, dp)) == -4
    e.decide_gps_batch_dev(d2.data_ptr(), 3, 90, [0, 1, 2], [0, 0, 0], nofix, 10.0, dp)
    e.decide_gps_batch_dev(d2.data_ptr(), 3, 90, [0, 1, 2], [0, 0, 0], None, 10.0, dp)
    # skipped and held frames ignore their fix, even without a table
    e.decide_gps_batch_dev(d2.data_ptr(), 3, 90, [0, 1, 2], [dc.FRAME_SKIP, dc.FRAME_HOLD, dc.FRAME_SKIP], fix, 10.0, dp)


def test_verification_after_a_gps_decision():
    """lcd_verify_decided_dev verifies the places a GPS decision accepted, and only those; lcd_process_fetch reports them."""
    import torch

    vocab = synth.make_binary_vocabulary(8192, 32, 1)
    wid = np.arange(1, 8193, dtype=np.int32)
    m = synth.make_map(wid, 400, 200, seed=2)
    st = synth.make_signature_store(vocab, wid, m)
    B = 32
    q, uv, places, _ = synth.make_query_frames_geo(st, m, B)
    eng = Engine(max_words=8192, max_signatures=402, max_queries=1000, max_batch=B)
    eng.add_words(wid, vocab)
    eng.last_word_id = 8192
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.sig_add_batch(m.sig_ids, st.desc, st.xyz)
    rng = np.random.default_rng(12)
    sig = [int(s) for s in m.sig_ids]
    fl = GpsFleet(B, dp=Engine.decide_params(loop_thr=0.11), eng=eng)
    fl.set_map(sig, *make_graph("chain", sig, n_levels(fl.text), rng))
    gps, off, pos = gc.trajectory_gps(len(sig), rng)
    fl.set_map_gps(gps, off)
    ns = len(sig)
    F = len(q) // B
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_uv = torch.from_numpy(uv.reshape(-1)).cuda()
    d_s = torch.from_numpy(m.sig_ids.astype(np.int32)).cuda()
    d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
    d_l = torch.zeros(B * ns, dtype=torch.float32, device="cuda")
    eng.localize_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), ns, ns + 1, d_w.data_ptr(), d_l.data_ptr())
    eng.synchronize()
    like = d_l.cpu().numpy().reshape(B, ns)
    # half the frames carry a fix on their true place, the other half a fix 2 km away (only the virtual place: nothing accepted)
    idx = {s: k for k, s in enumerate(sig)}
    fg = np.array([tuple(gps[idx[int(places[b])], :4]) + (5.0,) if b % 2 == 0 else gc.gps_row(pos[0][0] + 2000, pos[0][1]) for b in range(B)])
    dec, post, cmp = fl.step_gps(list(range(B)), like, np.zeros(B, np.int32), fg, 30.0, "gps decision")
    vp = Engine.verify_params(synth.CAMERA_K4)
    eng.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, vp)
    hyp, res = eng.process_fetch(B)
    accepted = [b for b in range(B) if dec[b]["status"] == dc.ACCEPTED]
    assert len(accepted) >= B // 4, dec["status"]
    for b in range(B):
        if b in accepted:
            h = int(dec[b]["loop_id"])
            v = eng.verify_batch(st.desc[h - 1][None], st.xyz[h - 1][None], q[b * F:(b + 1) * F][None], uv[b * F:(b + 1) * F][None],
                                 synth.CAMERA_K4)[0]
            assert res[b]["ok"] == v["ok"] and res[b]["n_inliers"] == len(v["inliers"]), f"frame {b}"
            assert hyp[b] == (h if v["ok"] else 0)
        else:
            assert not res[b]["ok"] and res[b]["n_matches"] == 0 and hyp[b] == 0, f"frame {b} was verified"
