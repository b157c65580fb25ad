"""The loop-closure decision of many localisation clients on the GPU (lcd_clients_* / lcd_decide_batch_dev / lcd_verify_decided_dev /
lcd_process_decide_batch_dev).

Posterior: per client against the sparse float restatement (oracle/bayes_py.py, pinned bit for bit to the reference's BayesFilter.cpp by
tests/test_oracle_bayes_ref.py) and, for a few clients, against the reference's compiled BayesFilter.cpp itself, each client with its own
filter.  Bar of tests/test_gpu_bayes_edges.py: rtol 1e-4, atol 1e-9, the same arg-max, the same virtual-place value.
Decisions: exactly those of the restated Rtabmap::process (oracle/decide_py.py) fed the GPU's own posterior and the client's state; against
the reference's posterior only where the value is farther than 1e-3 from every threshold."""
import numpy as np
import pytest

from bayes_cases import GRAPHS, PATTERNS, make_graph, n_levels, with_vp
from oracle import decide_py as dc
from oracle import oracle_py as orc
from oracle.bayes_py import BayesFilterOracle, parse_prediction_lc, prediction_columns
from rtabmap_b200 import Engine, LcdError, synth

pytestmark = pytest.mark.gpu

ACTIVE_MASK = dc.FRAME_SKIP | dc.FRAME_HOLD
MAX_BATCH = Engine.__init__.__defaults__[-1]  # the engine's default max_batch
UNTOUCHED = -7.0


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check_posterior(g, r, where):
    rel = float(np.max(np.abs(g - r) / np.maximum(np.abs(r), 1e-9)))
    assert np.allclose(g, r, rtol=1e-4, atol=1e-9), f"{where}: max rel {rel}"
    assert int(np.argmax(g)) == int(np.argmax(r)), f"{where}: argmax"
    assert abs(float(g[0]) - float(r[0])) <= 1e-4 * abs(float(r[0])) + 1e-9, f"{where}: virtual place"


def sparse_step(bf, ids, adj, cols):
    """One computePosterior of the sparse restatement: (posterior normalised by its float sum in id order, as the reference and the
    filter's kept state; the same normalised by the sum taken in double, as the kernel does)."""
    first = len(bf.posterior) == 0
    last = np.array([bf.posterior.get(i, np.float32(1 if first else 0)) for i in ids], np.float32)
    p = (np.asarray(adj, np.float32) * bf._prior(ids, last, *cols).astype(np.float32)).astype(np.float32)
    s = np.float32(p.astype(np.float64).sum())
    dsum = (p / s).astype(np.float32) if s != 0 else p
    return bf._update(ids, adj, lambda _: bf._prior(ids, last, *cols)), dsum


def check_float_sum(g, r, where):
    """Against a posterior normalised by a float sum over the places in id order.  Over thousands of places of similar value that sum
    drifts, which scales the whole posterior; the kernel sums in double.  Measured on an H100 80GB HBM3 (400 W power limit) with the
    flat adjusted likelihoods below: scales up to 1 + 1.5e-4 at 10 000 places and 1 + 1.1e-3 at 50 000, each one constant to 1e-5.
    Small maps: the bar itself.  Large maps: the same arg-max, and g / r one constant to 1e-5, within 5e-3 of 1."""
    if len(g) < 5000:
        return check_posterior(g, r, where)
    assert int(np.argmax(g)) == int(np.argmax(r)), f"{where}: argmax"
    k = r > 1e-30
    ratio = g[k].astype(np.float64) / r[k].astype(np.float64)
    assert ratio.max() - ratio.min() <= 1e-5 * ratio.mean(), f"{where}: not one scale ({ratio.min()}..{ratio.max()})"
    assert abs(ratio.mean() - 1.0) < 5e-3, f"{where}: scale {ratio.mean()}"


def raw_rows(rng, B, ns, heights=(0.3, 1.0, 4.0)):
    """Raw likelihood rows like Memory::computeLikelihood's: a noisy floor with a peak of varying height at a random place."""
    raw = (0.05 * rng.random((B, ns))).astype(np.float32)
    for b in range(B):
        k = int(rng.integers(ns))
        raw[b, k] = np.float32(heights[int(rng.integers(len(heights)))])
        if k + 1 < ns:
            raw[b, k + 1] = np.float32(0.5 * raw[b, k])
    return raw


def random_flags(rng, B):
    f = np.zeros(B, np.int32)
    u = rng.random(B)
    f[u < 0.1] = dc.FRAME_SKIP
    f[(u >= 0.1) & (u < 0.2)] = dc.FRAME_HOLD
    f[(u >= 0.2) & (u < 0.45)] = dc.FRAME_AGGRESSIVE
    return f


class Fleet:
    """One engine with n clients, and per client: the sparse restatement, optionally the compiled reference, the restated decision fed
    the GPU's posterior, and the restated decision fed the reference's posterior."""

    def __init__(self, n_clients, pattern="default", vpp=0.9, ref_clients=(), dp=None, eng=None):
        self.eng = eng or Engine()
        self.eng.clients_create(n_clients)
        self.n = n_clients
        self.text = PATTERNS[pattern]
        self.lc = parse_prediction_lc(self.text)
        self.vpp = vpp
        self.dp = dp or Engine.decide_params()
        kw = dict(loop_thr=self.dp.loop_thr, aggressive_loop_thr=self.dp.aggressive_loop_thr, loop_ratio=self.dp.loop_ratio,
                  max_loop_closure_distance=self.dp.max_loop_closure_distance)
        self.sparse = [BayesFilterOracle(self.text, vpp) for _ in range(n_clients)]
        self.refs = {k: orc.RefBayesFilter(self.text, vpp) for k in ref_clients} if orc.ref_bayes_lib() is not None else {}
        self.dec = [dc.DecideClient(**kw) for _ in range(n_clients)]
        self.dec_ref = {k: dc.DecideClient(**kw) for k in self.refs}
        self.statuses = set()

    def set_map(self, places, tables, stm):
        self.ids = with_vp(places, True)
        self.tables, self.stm = tables, stm
        cp, rows, lv = prediction_columns(self.ids, tables.__getitem__, stm)
        self.eng.clients_set_map(self.ids, cp, rows, lv, self.lc, self.vpp)
        self.cols = self.sparse[0].sparse_columns(self.ids, tables.__getitem__, stm)

    def reset(self, clients):
        self.eng.clients_reset(clients)
        for c in clients:
            self.sparse[c].reset()
            self.dec[c].reset()
            if c in self.refs:
                self.refs[c].reset()
                self.dec_ref[c].reset()

    def run(self, clients, raw, flags):
        """the GPU call alone: (decisions, posterior rows)"""
        import torch

        B, ns = raw.shape
        d_like = torch.from_numpy(np.ascontiguousarray(raw).reshape(-1)).cuda()
        d_post = torch.full((B * (ns + 1),), UNTOUCHED, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        self.eng.decide_batch_dev(d_like.data_ptr(), B, ns, clients, flags, self.dp, d_post.data_ptr())
        dec = self.eng.decide_fetch(B)
        return dec, d_post.cpu().numpy().reshape(B, ns + 1)

    def step(self, clients, raw, flags, where=""):
        clients = [int(c) for c in clients]
        dec, post = self.run(clients, raw, flags)
        adj = self.eng.adjust_likelihood(raw, self.dp.virtual_place_ratio)
        for b, c in enumerate(clients):
            w = f"{where} frame {b} client {c}"
            active = not flags[b] & ACTIVE_MASK
            if active:
                o, od = sparse_step(self.sparse[c], self.ids, adj[b], self.cols)
                check_posterior(post[b], od, w + " vs sparse restatement (double sum)")
                check_float_sum(post[b], o, w + " vs sparse restatement")
                if c in self.refs:
                    self.refs[c].set_graph(self.tables, self.stm)
                    r = self.refs[c].compute_posterior(self.ids, adj[b])
                    check_float_sum(post[b], r, w + " vs reference")
            else:
                assert (post[b] == np.float32(UNTOUCHED)).all(), w + ": a skipped / held frame's row was written"
            last = float(self.dec[c].highest[1])
            want = self.dec[c].decide(self.ids, post[b] if active else None, int(flags[b]))
            got = (int(dec[b]["highest_id"]), np.float32(dec[b]["highest_value"]), int(dec[b]["loop_id"]), int(dec[b]["status"]))
            assert got[0] == want[0] and bits(got[1]) == bits(want[1]) and got[2:] == want[2:], f"{w}: {got} != {want}"
            self.statuses.add(got[3])
            if c in self.refs:
                rd = self.dec_ref[c].decide(self.ids, r if active else None, int(flags[b]))
                # the highest real place: the same as on the reference's posterior unless its top two real places are a near-tie
                tie = False
                if active and len(r) > 2:
                    top = np.sort(r[1:].astype(np.float64))[-2:]
                    tie = top[1] - top[0] <= 1e-4 * top[1]
                if not tie:
                    assert rd[0] == want[0], f"{w}: highest real place {want[0]}, on the reference posterior {rd[0]}"
                thr = (self.dp.loop_thr, self.dp.aggressive_loop_thr, self.dp.loop_ratio * last)
                if not tie and all(abs(float(want[1]) - t) > 1e-3 for t in thr):
                    assert rd[2:] == want[2:], f"{w}: decision on the reference posterior {rd} != {want}"
                self.dec_ref[c].highest = self.dec[c].highest   # follow the GPU's state, so that one near-threshold frame does not spread
        return dec, post


VPP = (0.9, 0.0, 1.0)   # Bayes/VirtualPlacePriorThr: the virtual-place row and column of every branch (vpp, 1/n, and P[r][0] = 0)
CASES = [(p, GRAPHS[i % len(GRAPHS)], (1, 2, 33, 128, MAX_BATCH)[i % 5], VPP[i % 3]) for i, p in enumerate(PATTERNS)] + [
    ("default", "hub", 2, 0.0), ("trunc5", "loops", MAX_BATCH, 1.0), ("sum1", "merged", 128, 0.9)]


@pytest.mark.parametrize("pattern,graph,n_clients,vpp", CASES)
def test_posterior_and_decisions_over_twenty_steps(pattern, graph, n_clients, vpp):
    """Twenty steps over a map of a few hundred places that grows every fifth step; every client in every step (some skipped or held),
    in a shuffled order; two clients also against the reference's own BayesFilter.cpp."""
    rng = np.random.default_rng(sum(map(ord, f"{pattern} {graph} {n_clients}")))
    dp = Engine.decide_params(loop_thr=0.11, loop_ratio=0.5 if n_clients % 2 else 0.0)
    fl = Fleet(n_clients, pattern, vpp=vpp, ref_clients=(0, n_clients - 1), dp=dp)
    places = list(range(1, 301))
    for t in range(20):
        if t % 5 == 0:
            places = places + [places[-1] + 1, places[-1] + 2]
            fl.set_map(places, *make_graph(graph, places, n_levels(fl.text), rng))
        order = rng.permutation(n_clients)
        fl.step(order, raw_rows(rng, n_clients, len(places)), random_flags(rng, n_clients), f"{pattern} {graph} B={n_clients} step {t}")
    assert dc.ACCEPTED in fl.statuses


@pytest.mark.parametrize("n", [10000, 50000])
def test_large_maps_128_clients(n):
    """128 clients against the sparse restatement at 10 000 and 50 000 places; at 10 000, two clients against the reference too."""
    rng = np.random.default_rng(n)
    fl = Fleet(128, "trunc5", ref_clients=(5, 77) if n <= 10000 else ())
    places = list(range(1, n + 1))
    fl.set_map(places, *make_graph("chain", places, n_levels(fl.text), rng))
    for t in range(2):
        fl.step(rng.permutation(128), raw_rows(rng, 128, n), random_flags(rng, 128), f"n={n} step {t}")


def test_every_status_and_flag():
    """Thresholds, ratio and the single-hypothesis map chosen so that every status of the decision occurs, each checked exactly."""
    rng = np.random.default_rng(3)
    places = list(range(1, 41))
    seen = set()
    for dp in (Engine.decide_params(loop_thr=0.11, loop_ratio=0.9), Engine.decide_params(loop_thr=0.6, aggressive_loop_thr=0.3, loop_ratio=0.0),
               Engine.decide_params(loop_thr=0.11, virtual_place_ratio=1)):
        fl = Fleet(16, dp=dp)
        fl.set_map(places, *make_graph("loops", places, n_levels(fl.text), rng))
        for t in range(12):
            raw = raw_rows(rng, 16, 40, heights=(0.06, 0.2, 1.0, 5.0))
            raw[t % 16] = 0          # no place scores at all
            fl.step(rng.permutation(16), raw, random_flags(rng, 16), f"step {t}")
        seen |= fl.statuses
    single = Fleet(3, dp=Engine.decide_params(loop_thr=0.11))
    single.set_map([7], {7: {7: 0}}, [])
    single.step([0, 1, 2], np.array([[0.5], [2.0], [0.0]], np.float32), np.zeros(3, np.int32), "one real place")
    assert dc.SINGLE_HYPOTHESIS in single.statuses
    # LCD_DECIDE_NO_HYPOTHESIS needs a posterior of 0 on every real place: adjustLikelihood never outputs 0 and every real place's prior
    # is > 0 once it has a last posterior, so valid inputs do not reach it; its branch is the restatement's, checked on every frame
    want = {dc.SKIPPED, dc.HELD, dc.UNDER_THRESHOLD, dc.UNDER_RATIO, dc.SINGLE_HYPOTHESIS, dc.RATIO, dc.LAST_NULL, dc.ACCEPTED}
    assert want <= seen | single.statuses, f"statuses not reached: {want - seen}"


def test_a_client_gets_the_same_bits_alone_anywhere_in_a_batch_and_in_every_run():
    rng = np.random.default_rng(8)
    places = list(range(1, 2001))
    tables, stm = make_graph("loops", places, n_levels(PATTERNS["default"]), rng)
    steps = [(raw_rows(rng, 128, 2000), random_flags(rng, 128)) for _ in range(3)]
    track = 9
    runs = []
    for B, pos, run in [(1, 0, 0), (128, 0, 0), (128, 77, 0), (128, 127, 0), (128, 77, 1), (33, 32, 0)]:
        fl = Fleet(128)
        fl.set_map(places, tables, stm)
        out = []
        for t, (raw, flags) in enumerate(steps):
            others = [c for c in np.random.default_rng(100 * t + pos + run).permutation(128) if c != track][:B - 1]
            clients = others[:pos] + [track] + others[pos:]
            rows = np.random.default_rng(t + 7 * run).permutation(raw)[:B].copy()
            rows[pos] = raw[0]
            fr = np.random.default_rng(t + 11 * run).permutation(flags)[:B].copy()
            fr[pos] = 0 if t != 1 else dc.FRAME_AGGRESSIVE
            dec, post = fl.run(clients, rows, fr)
            out.append((bits(post[pos]).copy(), dec[pos].tobytes()))
        runs.append(out)
    for r in runs[1:]:
        for t in range(3):
            assert np.array_equal(r[t][0], runs[0][t][0]), f"step {t}: posterior bits differ"
            assert r[t][1] == runs[0][t][1], f"step {t}: decision differs"


def test_map_changes_rekey_like_the_reference_and_reset_of_one_client():
    """Places are added, removed and re-added between steps; client 2 computes nothing across two set_map calls and must keep the value of
    a place that left and came back, as the reference's updatePosterior does; client 4 is reset among the others."""
    if orc.ref_bayes_lib() is None:
        pytest.skip("the reference's BayesFilter.cpp is not built")
    rng = np.random.default_rng(21)
    fl = Fleet(6, ref_clients=range(6), dp=Engine.decide_params(loop_thr=0.11, loop_ratio=0.3))
    levels = n_levels(fl.text)
    base = list(range(1, 151))
    maps = [base, base + [151, 152], [p for p in base if p not in (40, 41, 90)] + [151, 152, 153],
            [p for p in base if p != 90] + [151, 152, 153, 154], base[:120]]
    for t, places in enumerate(maps):
        fl.set_map(places, *make_graph("loops", places, levels, rng))
        clients = [0, 1, 3, 4, 5] if t in (1, 2) else list(range(6))
        if t == 3:
            fl.reset([4])
        raw = raw_rows(rng, len(clients), len(places))
        flags = np.zeros(len(clients), np.int32)
        if t == 4:
            flags[1] = dc.FRAME_HOLD
        fl.step(clients, raw, flags, f"map {t}")


def test_a_failed_set_map_leaves_the_previous_map_in_place():
    """A map whose client posteriors do not fit on the device is refused with LCD_ERR_CAPACITY after its tables were built; the clients
    then go on against the previous map exactly as on an engine that never saw the call."""
    import torch

    n_clients, n_big = 25000, 1000000     # 25 000 x 1 000 001 floats = 100 GB of posteriors: more than the card holds
    rng = np.random.default_rng(31)
    places = list(range(1, 101))
    tables, stm = make_graph("loops", places, n_levels(PATTERNS["default"]), rng)
    ids = with_vp(places, True)
    cp, rows, lv = prediction_columns(ids, tables.__getitem__, stm)
    lc = parse_prediction_lc(PATTERNS["default"])
    engines = [Engine(), Engine()]
    for e in engines:
        e.clients_create(n_clients)
        e.clients_set_map(ids, cp, rows, lv, lc, 0.9)
    big_ids = np.concatenate([[-1], np.arange(1, n_big + 1)]).astype(np.int32)
    big_cp = np.concatenate([[0, 0], np.arange(1, n_big + 1)]).astype(np.int64)   # every place lists only itself
    clients = [3, 24999, 7]
    dp = Engine.decide_params(loop_thr=0.11, loop_ratio=0.5)
    out = []
    for k, e in enumerate(engines):
        got = []
        for t in range(3):
            if k == 0 and t == 1:
                with pytest.raises(LcdError) as ex:
                    e.clients_set_map(big_ids, big_cp, np.arange(1, n_big + 1, dtype=np.int32), np.zeros(n_big, np.int32), lc, 0.9)
                assert ex.value.code == -3
            raw = raw_rows(np.random.default_rng(t), len(clients), 100)
            d_like = torch.from_numpy(raw.reshape(-1)).cuda()
            d_post = torch.zeros(len(clients) * 101, dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            e.decide_batch_dev(d_like.data_ptr(), len(clients), 100, clients, [0, 0, 0], dp, d_post.data_ptr())
            got.append((e.decide_fetch(len(clients)).tobytes(), bits(d_post.cpu().numpy()).copy()))
        out.append(got)
    for t in range(3):
        assert out[0][t][0] == out[1][t][0] and np.array_equal(out[0][t][1], out[1][t][1]), f"step {t}"


@pytest.fixture(scope="module")
def c2_store():
    vocab = synth.make_binary_vocabulary(49152, 32, 1)
    ids = np.arange(1, 49153, dtype=np.int32)
    m = synth.make_map(ids, 10000, 200, seed=2)
    st = synth.make_signature_store(vocab, ids, m)
    q, uv, places, poses = synth.make_query_frames_geo(st, m, 128)
    eng = Engine(max_words=49152, max_signatures=10002, max_queries=1000, max_batch=128)
    eng.add_words(ids, vocab)
    eng.last_word_id = 49152
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.sig_add_batch(m.sig_ids, st.desc, st.xyz)
    return eng, m, st, q, uv, places


def test_fused_call_at_c2_scale(c2_store):
    """128 frames against 10 000 places with the signature store: word ids and likelihood equal lcd_localize_batch_dev bit for bit, the
    decisions equal adjustLikelihood + the per-client restatement, every accepted frame's verification equals lcd_verify_batch of the
    same (loop id, frame) pair, frames that were not accepted are not verified, and a failed registration / a long transform reject."""
    import torch

    eng, m, st, q, uv, places = c2_store
    B, ns = 128, len(m.sig_ids)
    F = len(q) // B
    rng = np.random.default_rng(4)
    fl = Fleet(B, dp=Engine.decide_params(loop_thr=0.11), eng=eng)
    sig = [int(s) for s in m.sig_ids]
    fl.set_map(sig, *make_graph("chain", sig, n_levels(fl.text), rng))
    vp = Engine.verify_params(synth.CAMERA_K4)
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_uv = torch.from_numpy(uv.reshape(-1)).cuda()
    d_s = torch.from_numpy(m.sig_ids.astype(np.int32)).cuda()
    removed = [int(places[b]) for b in (20, 21, 22)]   # their store rows go: an accepted hypothesis there fails registration
    for s in removed:
        eng.sig_remove(s)
    flags = np.zeros(B, np.int32)
    flags[:4] = dc.FRAME_SKIP
    flags[4:8] = dc.FRAME_HOLD
    flags[8:40] = dc.FRAME_AGGRESSIVE
    clients = rng.permutation(B)
    norms = None
    for step, max_dist in enumerate((0.0, None)):
        if max_dist is None:                            # second step: a distance limit under some accepted transforms' norms
            max_dist = float(np.median(norms))
        fl.dp = Engine.decide_params(loop_thr=0.11, max_loop_closure_distance=max_dist)
        for k in range(B):
            fl.dec[k].max_loop_closure_distance = np.float32(max_dist)
        d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
        d_l = torch.zeros(B * ns, dtype=torch.float32, device="cuda")
        d_p = torch.full((B * (ns + 1),), UNTOUCHED, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        eng.process_decide_batch_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, ns, ns + 1, vp, clients, flags, fl.dp, d_w.data_ptr(), d_l.data_ptr(),
                                     d_p.data_ptr())
        dec = eng.decide_fetch(B)
        hyp, res = eng.process_fetch(B)
        words, like, post = d_w.cpu().numpy(), d_l.cpu().numpy().reshape(B, ns), d_p.cpu().numpy().reshape(B, ns + 1)
        # quantise + score: lcd_localize_batch_dev with the map's ids
        d_w2 = torch.zeros(B * F, dtype=torch.int32, device="cuda")
        d_l2 = torch.zeros(B * ns, dtype=torch.float32, device="cuda")
        eng.localize_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), ns, ns + 1, d_w2.data_ptr(), d_l2.data_ptr())
        eng.synchronize()
        assert np.array_equal(words, d_w2.cpu().numpy()) and np.array_equal(bits(like), bits(d_l2.cpu().numpy().reshape(B, ns)))
        # decisions: adjust + the per-client restatement on the GPU posterior, then the verification rules
        adj = eng.adjust_likelihood(like)
        acc = []
        for b in range(B):
            c = int(clients[b])
            active = not flags[b] & ACTIVE_MASK
            if active:
                o, od = sparse_step(fl.sparse[c], fl.ids, adj[b], fl.cols)
                check_posterior(post[b], od, f"step {step} frame {b}")
                check_float_sum(post[b], o, f"step {step} frame {b}")
            want = fl.dec[c].decide(fl.ids, post[b] if active else None, int(flags[b]))
            r = res[b]
            if want[3] == dc.ACCEPTED:
                h = want[2]
                v = eng.verify_batch(st.desc[h - 1][None], st.xyz[h - 1][None], q[b * F:(b + 1) * F][None], uv[b * F:(b + 1) * F][None],
                                     synth.CAMERA_K4, n_from=[0 if h in removed else st.desc.shape[1]])[0]
                assert r["ok"] == v["ok"] and r["n_matches"] == len(v["matches"]) and r["n_inliers"] == len(v["inliers"]), f"frame {b}"
                if v["ok"]:
                    assert np.array_equal(r["rvec"], v["rvec"]) and np.array_equal(r["tvec"], v["tvec"]), f"frame {b}"
                t = v["transform"]
                want = fl.dec[c].verified(want, v["ok"], (t[0, 3], t[1, 3], t[2, 3]))
                if v["ok"]:
                    acc.append(float(np.linalg.norm(t[:, 3])))
            else:
                assert not r["ok"] and r["n_matches"] == 0, f"frame {b} was verified without an accepted hypothesis"
            got = (int(dec[b]["highest_id"]), np.float32(dec[b]["highest_value"]), int(dec[b]["loop_id"]), int(dec[b]["status"]))
            assert got[0] == want[0] and bits(got[1]) == bits(want[1]) and got[2:] == want[2:], f"step {step} frame {b}: {got} != {want}"
            assert hyp[b] == got[2]
            fl.statuses.add(got[3])
        norms = acc
        assert len(acc) >= B // 4, f"only {len(acc)} registered loop closures"
    assert {dc.SKIPPED, dc.HELD, dc.ACCEPTED, dc.VERIFY_REJECTED, dc.DISTANCE_REJECTED} <= fl.statuses, fl.statuses


def test_errors():
    import torch

    eng = Engine()
    dp = Engine.decide_params()
    d = torch.zeros(64, dtype=torch.float32, device="cuda")
    lc = parse_prediction_lc(PATTERNS["default"])

    def code(f):
        with pytest.raises(LcdError) as ex:
            f()
        return ex.value.code

    assert code(lambda: eng.decide_batch_dev(d.data_ptr(), 1, 3, [0], [0], dp)) == -4              # no clients
    eng.clients_create(4)
    assert code(lambda: eng.decide_batch_dev(d.data_ptr(), 1, 3, [0], [0], dp)) == -4              # no map
    ids = [-1, 1, 2, 3]
    cp, rows, lv = prediction_columns(ids, {1: {1: 0, 2: 1}, 2: {1: 1, 2: 0, 3: 1}, 3: {2: 1, 3: 0}}.__getitem__)
    assert code(lambda: eng.clients_set_map(ids[1:], *prediction_columns(ids[1:], {1: {1: 0}, 2: {2: 0}, 3: {3: 0}}.__getitem__), lc)) == -1
    assert code(lambda: eng.clients_set_map(ids, cp, rows, lv, [0.1])) == -1
    eng.clients_set_map(ids, cp, rows, lv, lc)
    assert code(lambda: eng.decide_batch_dev(d.data_ptr(), 2, 3, [1, 1], [0, 0], dp)) == -1          # repeated client
    assert code(lambda: eng.decide_batch_dev(d.data_ptr(), 1, 3, [4], [0], dp)) == -1                # out of range
    assert code(lambda: eng.decide_batch_dev(d.data_ptr(), 1, 3, [-1], [0], dp)) == -1
    assert code(lambda: eng.decide_batch_dev(d.data_ptr(), 1, 4, [0], [0], dp)) == -1                # ns != the map's real places
    for bad in (dict(loop_thr=-0.1), dict(loop_thr=1.5), dict(aggressive_loop_thr=float("nan")), dict(loop_ratio=2.0),
                dict(max_loop_closure_distance=-1.0), dict(virtual_place_ratio=2)):
        assert code(lambda: eng.decide_batch_dev(d.data_ptr(), 1, 3, [0], [0], Engine.decide_params(**bad))) == -1, bad
    assert code(lambda: eng.clients_reset([9])) == -1
    assert code(lambda: eng.decide_fetch(1)) == -4                                                    # nothing decided yet
    # verification of a decision: none yet, then with the store empty
    vocab = synth.make_binary_vocabulary(500, 32, 1)
    wid = np.arange(1, 501, dtype=np.int32)
    m = synth.make_map(wid, 3, 60, seed=2)
    st = synth.make_signature_store(vocab, wid, m)
    eng.add_words(wid, vocab)
    eng.last_word_id = 500
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    vp = Engine.verify_params(synth.CAMERA_K4)
    dq = torch.zeros(60 * 32, dtype=torch.uint8, device="cuda")
    duv = torch.zeros(60 * 2, dtype=torch.float32, device="cuda")
    eng.sig_add_batch(m.sig_ids, st.desc, st.xyz)
    assert code(lambda: eng.verify_decided_dev(dq.data_ptr(), duv.data_ptr(), 1, 60, vp)) == -4
    eng.decide_batch_dev(d.data_ptr(), 1, 3, [0], [0], dp)
    eng.verify_decided_dev(dq.data_ptr(), duv.data_ptr(), 1, 60, vp)
    assert code(lambda: eng.verify_decided_dev(dq.data_ptr(), duv.data_ptr(), 2, 60, vp)) == -1        # not the decision's frame count
    eng.verify_top_dev(dq.data_ptr(), duv.data_ptr(), 1, 60, d.data_ptr(), torch.tensor([1, 2, 3], dtype=torch.int32, device="cuda").data_ptr(), 3, vp)
    assert code(lambda: eng.verify_decided_dev(dq.data_ptr(), duv.data_ptr(), 1, 60, vp)) == -4        # the arg-max replaced the hypotheses
    # fused call: sharded engine and float engine
    eng.shard_set_row_offset(64)
    assert code(lambda: eng.process_decide_batch_dev(dq.data_ptr(), duv.data_ptr(), 1, 60, 3, 4, vp, [0], [0], dp)) == -4
    f = Engine(desc_type=1, desc_dim=64)
    f.clients_create(1)
    f.clients_set_map(ids, cp, rows, lv, lc)
    assert code(lambda: f.process_decide_batch_dev(dq.data_ptr(), duv.data_ptr(), 1, 60, 3, 4, vp, [0], [0], dp)) == -1
    f.decide_batch_dev(d.data_ptr(), 1, 3, [0], [0], dp)     # the decision itself serves float engines
    assert f.decide_fetch(1)["status"][0] in range(11)
