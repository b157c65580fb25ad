"""The batched localisation decision on float-descriptor engines (LCD_DESC_F32, 64-D and 128-D), the composition float clients use:
lcd_localize_batch_dev -> lcd_decide_batch_dev -> lcd_verify_decided_dev, and lcd_decide_proximity_dev.

Decisions: exactly those of the restated Rtabmap::process (oracle/decide_py.py) fed the GPU's posterior, then the verification rules on
the oracle's registration (tests/test_gpu_decide.py's Fleet).  Proximity: candidates, keys, paths and decisions as the restatement of
oracle/proximity_py.py (tests/test_gpu_proximity.py's run and check).  Every registration: lcd_verify_batch on the same (place, frame)
pair bit for bit, and the CPU oracle.  The scenes include frames whose accepted place has no store row (a removed signature, or a
proximity candidate past the store) and frames whose registration fails."""
import numpy as np
import pytest

from bayes_cases import make_graph, n_levels
from oracle import decide_py as dc
from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import LCD_DESC_F32
from test_gpu_decide import Fleet
from test_gpu_proximity import F, S, check as px_check, run as px_run, scene as px_scene, set_map as px_set_map
from test_gpu_verify_f32 import IMG, K4, WIN, assert_oracle, assert_same_bits, near, rand_desc

pytestmark = pytest.mark.gpu

N_WORDS = 3000
N_FRAMES = 128


@pytest.fixture(scope="module", params=[64, 128])
def fworld(request):
    """(dim, vocab, word ids, map, store, frame descriptors [N_FRAMES*F, dim], uv, place of every frame): S places of F features, each
    feature a near copy of a dictionary word; frame b re-observes place places[b] from a nearby pose, 20 % of its features replaced by
    unrelated descriptors at random pixels."""
    dim = request.param
    vocab = synth.make_float_vocabulary(N_WORDS, dim, 1)
    wid = np.arange(1, N_WORDS + 1, dtype=np.int32)
    m = synth.make_map(wid, S, F, seed=2)
    rng = np.random.default_rng(4 + dim)
    desc = near(rng, vocab[m.sig_words.reshape(-1) - 1], 0.2).reshape(S, F, dim)
    xyz = np.empty((S, F, 3), np.float32)
    z = rng.uniform(0.5, 5.0, (S, F)).astype(np.float32)
    xyz[..., 0] = rng.uniform(-0.55, 0.55, (S, F)).astype(np.float32) * z
    xyz[..., 1] = rng.uniform(-0.40, 0.40, (S, F)).astype(np.float32) * z
    xyz[..., 2] = z
    xyz[rng.random((S, F)) < 0.02] = np.nan
    places = rng.integers(0, S, N_FRAMES)
    q = np.empty((N_FRAMES, F, dim), np.float32)
    uv = np.empty((N_FRAMES, F, 2), np.float32)
    for b, p in enumerate(places):
        perm = rng.permutation(F)
        q[b] = near(rng, desc[p][perm], 0.4)
        X = np.nan_to_num(xyz[p][perm].astype(np.float64), nan=1.0)
        uv[b] = orc.project_points(X, K4, rng.normal(0, 0.06, 3), rng.normal(0, 0.1, 3)) + rng.normal(0, 0.5, (F, 2))
        out = rng.permutation(F)[:F // 5]
        q[b, out] = rand_desc(rng, len(out), dim)
        uv[b, out] = np.stack([rng.uniform(0, 640, len(out)), rng.uniform(0, 480, len(out))], 1)
    return dim, vocab, wid, m, synth.SynthStore(desc, xyz), q.reshape(-1, dim), uv.reshape(-1, 2), m.sig_ids[places]


def make_engine(fworld, n_places, n_clients):
    dim, vocab, wid, m, st, *_ = fworld
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=dim, max_words=N_WORDS, max_signatures=n_places + 2, max_queries=F, max_batch=128)
    eng.add_words(wid, vocab)
    eng.last_word_id = N_WORDS
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.sig_add_batch(m.sig_ids, st.desc, st.xyz)
    eng.clients_create(n_clients)
    return eng


def test_localize_decide_verify_decided(fworld):
    """lcd_localize_batch_dev -> lcd_decide_batch_dev -> lcd_verify_decided_dev for 48 clients, the second pass on: skipped, held and
    aggressive frames; accepted places whose signature was removed (no store row: the registration fails); a second step with
    RGBD/MaxLoopClosureDistance at the median of the first step's translations."""
    import torch

    dim, vocab, wid, m, st, q, uv, places = fworld
    B, ns = 48, S
    eng = make_engine(fworld, S, B)
    rng = np.random.default_rng(5)
    fl = Fleet(B, dp=Engine.decide_params(loop_thr=0.11), eng=eng)
    sig = [int(s) for s in m.sig_ids]
    fl.set_map(sig, *make_graph("chain", sig, n_levels(fl.text), rng))
    removed = {int(places[b]) for b in (3, 4)}
    for s in removed:
        eng.sig_remove(s)
    vp = Engine.verify_params(K4, image_size=IMG, repeat_once=True, guess_win_size=WIN)
    d_q = torch.from_numpy(np.ascontiguousarray(q[:B * F]).reshape(-1)).cuda()
    d_uv = torch.from_numpy(np.ascontiguousarray(uv[:B * F]).reshape(-1)).cuda()
    d_s = torch.from_numpy(m.sig_ids.astype(np.int32)).cuda()
    flags = np.zeros(B, np.int32)
    flags[:3] = dc.FRAME_SKIP
    flags[5:8] = dc.FRAME_HOLD
    flags[8:20] = dc.FRAME_AGGRESSIVE
    clients = rng.permutation(B)
    vb = Engine(desc_type=LCD_DESC_F32, desc_dim=dim)
    w_ref, l_ref = eng.localize_batch(q[:B * F], B, m.sig_ids, ns + 1)
    norms, n_removed = None, 0
    for step, max_dist in enumerate((0.0, None)):
        if max_dist is None:
            max_dist = float(np.median(norms))
        fl.dp = Engine.decide_params(loop_thr=0.11, max_loop_closure_distance=max_dist)
        for k in range(B):
            fl.dec[k].max_loop_closure_distance = np.float32(max_dist)
        d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
        d_l = torch.zeros(B * ns, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        eng.localize_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), ns, ns + 1, d_w.data_ptr(), d_l.data_ptr())
        eng.synchronize()
        like = d_l.cpu().numpy().reshape(B, ns)
        assert np.array_equal(d_w.cpu().numpy().reshape(B, F), w_ref) and np.array_equal(like.view(np.uint32), l_ref.view(np.uint32))
        dec, _ = fl.step(clients, like, flags, f"step {step}")   # decisions and posterior against the restatement
        eng.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, vp)
        hyp, res = eng.process_fetch(B)
        final = eng.decide_fetch(B)
        acc = []
        for b in range(B):
            c = int(clients[b])
            want = (int(dec[b]["highest_id"]), np.float32(dec[b]["highest_value"]), int(dec[b]["loop_id"]), int(dec[b]["status"]))
            r = res[b]
            if want[3] == dc.ACCEPTED:
                h = want[2]
                n_from = 0 if h in removed else F
                n_removed += h in removed
                d, x = st.desc[h - 1][:n_from], st.xyz[h - 1][:n_from]
                fq, fu = q[b * F:(b + 1) * F], uv[b * F:(b + 1) * F]
                g = vb.verify_batch(st.desc[h - 1][None], st.xyz[h - 1][None], fq[None], fu[None], K4, n_from=[n_from], image_size=IMG,
                                    repeat_once=True, guess_win_size=WIN)[0]
                assert_same_bits(r, g, (step, b))
                o = orc.verify_pair_repeat(d, x, fq, fu, K4, image_size=IMG, guess_win_size=WIN)
                assert_oracle(r, o, (step, b))
                t = o["transform"]
                want = fl.dec[c].verified(want, o["ok"], (t[0, 3], t[1, 3], t[2, 3]))
                if o["ok"]:
                    acc.append(float(np.linalg.norm(t[:, 3])))
            else:
                assert not r["ok"] and r["n_matches"] == 0, f"frame {b} was registered without an accepted hypothesis"
            got = (int(final[b]["highest_id"]), np.float32(final[b]["highest_value"]), int(final[b]["loop_id"]), int(final[b]["status"]))
            assert got[0] == want[0] and got[1].tobytes() == want[1].tobytes() and got[2:] == want[2:], f"step {step} frame {b}: {got} != {want}"
            assert hyp[b] == got[2]
            fl.statuses.add(got[3])
        norms = acc
        assert len(acc) >= B // 4, f"only {len(acc)} registered loop closures"
    assert n_removed >= 1, n_removed
    assert {dc.SKIPPED, dc.HELD, dc.ACCEPTED, dc.VERIFY_REJECTED, dc.DISTANCE_REJECTED} <= fl.statuses, fl.statuses
    vb.close()
    eng.close()


def test_proximity_detection(fworld):
    """lcd_decide_proximity_dev on 1000 places, 37 clients: candidates, keys, paths and decisions as the restatement; every attempted
    registration (store row through its slot, frame row read in place) as lcd_verify_batch bit for bit and the oracle.  The signatures
    of three frames' own places are removed first: those candidates have no store row and are not registered."""
    dim, *world = fworld
    vocab, wid, m, st, q, uv, places = world
    n_places, B = 1000, 37
    ids, poses, nbr, ptr, flat = px_scene(n_places)
    eng = make_engine(fworld, n_places, B)
    removed = {int(places[b]) for b in (0, 3, 6)}
    for s in removed:
        eng.sig_remove(s)
    px_set_map(eng, ids)
    eng.clients_set_map_poses(ids, poses, ptr, flat)
    out = px_run(eng, world, ids, poses, B, seed=n_places + B)
    statuses = px_check(world, ids, poses, nbr, out, check_verify=False)
    assert dc.ACCEPTED in statuses and ("suppressed", True) in statuses and ("suppressed", False) in statuses, statuses
    vb = Engine(desc_type=LCD_DESC_F32, desc_dim=dim)
    n_checked = n_ok = n_absent = 0
    for b, o in enumerate(out["order"]):
        fq, fu = q[o * F:(o + 1) * F], uv[o * F:(o + 1) * F]
        for g in out["rec"][b]["paths"]:
            h, r = g["candidate_id"], g["result"]
            if h > S:
                assert not r["ok"] and r["n_matches"] == 0, (b, h)
                continue
            n_from = 0 if h in removed else F
            n_absent += h in removed
            v = vb.verify_batch(st.desc[h - 1][None], st.xyz[h - 1][None], fq[None], fu[None], K4, n_from=[n_from])[0]
            assert_same_bits(r, v, (b, h))
            assert_oracle(r, orc.verify_pair_cov(st.desc[h - 1][:n_from], st.xyz[h - 1][:n_from], fq, fu, K4), (b, h))
            n_checked += 1
            n_ok += r["ok"]
    assert n_checked >= 20 and n_ok >= 5 and n_absent >= 1, (n_checked, n_ok, n_absent)
    vb.close()
    eng.close()
