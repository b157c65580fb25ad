"""The similarity likelihood (Memory::computeLikelihood with Kp/TfIdfLikelihoodUsed=false) on the GPU against the CPU oracle
(oracle/similarity_py.py): word pairs bit for bit, global-descriptor values within the fp32 summation bound of the exact dot
product and bit-identical across batch sizes, frame positions, entry points and runs."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from oracle import similarity_py as sim
from rtabmap_b200 import Engine, LcdError, synth

pytestmark = pytest.mark.gpu

EXTRA_IDS = np.array([0, -3, 10005, 99999], np.int32)  # virtual place, a negative id, ids the index does not know


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def word_likelihood(frame_words, ids, sig_words):
    """Vectorised oracle of the word branch: sig_words maps id -> int array of its words; same rules as sim.compare_to."""
    nvalid = {s: int((np.asarray(w) > 0).sum()) for s, w in sig_words.items()}
    out = np.zeros((len(frame_words), len(ids)), np.float32)
    counts = {s: dict(zip(*np.unique(np.asarray(w)[np.asarray(w) > 0], return_counts=True))) for s, w in sig_words.items()}
    for f, fw in enumerate(frame_words):
        fw = np.asarray(fw)
        uq, cq = np.unique(fw[fw > 0], return_counts=True)
        qd = dict(zip(uq.tolist(), cq.tolist()))
        nq = int((fw > 0).sum())
        for k, s in enumerate(ids):
            s = int(s)
            if s <= 0 or nq == 0 or nvalid.get(s, 0) == 0:
                continue
            c = counts[s]
            pairs = sum(min(n, c.get(w, 0)) for w, n in qd.items()) if len(qd) < len(c) else sum(min(n, qd.get(w, 0)) for w, n in c.items())
            out[f, k] = np.float32(pairs) / np.float32(max(nq, nvalid[s]))
    return out


def csr_likelihood(frame_words, ids, m):
    """The same over the CSR map of synth.make_map (fast at C2 scale): pairs through the word -> (signature, count) lists."""
    S = int(m.sig_ids.max()) + 1
    nvalid = np.bincount(m.sig, weights=m.cnt, minlength=S).astype(np.int64)
    out = np.zeros((len(frame_words), len(ids)), np.float32)
    ids = np.asarray(ids)
    known = (ids > 0) & (ids < S)
    for f, fw in enumerate(frame_words):
        fw = np.asarray(fw)
        uq, cq = np.unique(fw[fw > 0], return_counts=True)
        idx = np.searchsorted(m.word_ids, uq)
        ok = idx < len(m.word_ids)
        ok[ok] = m.word_ids[idx[ok]] == uq[ok]
        idx, cq = idx[ok], cq[ok]
        st, ln = m.row_ptr[idx], m.row_ptr[idx + 1] - m.row_ptr[idx]
        pos = np.repeat(st - np.cumsum(ln) + ln, ln) + np.arange(int(ln.sum()))
        pairs = np.bincount(m.sig[pos], weights=np.minimum(np.repeat(cq, ln), m.cnt[pos]), minlength=S).astype(np.int64)
        nq = int((fw > 0).sum())
        kk = np.nonzero(known)[0]
        s = ids[kk]
        den = np.maximum(nq, nvalid[s])
        v = pairs[s].astype(np.float32) / den.astype(np.float32)
        v[(nvalid[s] == 0) | (nq == 0)] = 0
        out[f, kk] = v
    return out


def unit(rng, n, d):
    g = rng.normal(size=(n, d)).astype(np.float32)
    return (g / np.linalg.norm(g, axis=1, keepdims=True)).astype(np.float32)


def assert_gdesc_close(like, Q, G):
    """every value within the bound of an exact dot product; exact = fsum per pair (small) or float64 BLAS plus its own error."""
    q64, g64 = Q.astype(np.float64), G.astype(np.float64)
    dot = q64 @ g64.T
    absd = np.abs(q64) @ np.abs(g64).T
    D = Q.shape[1]
    tol = sim.gamma(D) * absd / 2 + 2 * D * 2.0 ** -53 * absd + np.spacing(np.abs(like).astype(np.float32)).astype(np.float64)
    err = np.abs(like.astype(np.float64) - (dot + 1.0) / 2.0)
    assert np.all(err <= tol), f"max err {err.max()} vs tol {tol[np.unravel_index(err.argmax(), err.shape)]}"


# ------------------------------------------------------------------------------------------------ C2 scale ---------
@pytest.fixture(scope="module")
def c2():
    vocab = synth.make_binary_vocabulary(49152, 32, 1)
    ids = np.arange(1, 49153, dtype=np.int32)
    m = synth.make_map(ids, 10000, 200, seed=2)
    eng = Engine(max_words=49152, max_signatures=10002, max_queries=1000, max_batch=128)
    eng.add_words(ids, vocab)
    eng.last_word_id = 49152
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    q, places = synth.make_query_frames(vocab, ids, m, 128, 1000, seed=3)
    return eng, vocab, ids, m, q, places


@pytest.mark.parametrize("incremental", [True, False])
def test_word_pairs_bit_exact_at_c2_scale(c2, incremental):
    import torch

    eng, vocab, ids, m, q, places = c2
    B, F = 128, 1000
    sig_list = np.concatenate([m.sig_ids[:5000], EXTRA_IDS, m.sig_ids[5000:]]).astype(np.int32)
    words, like = eng.localize_similarity_batch(q, B, sig_list, incremental=incremental)
    # the quantise half is localize_batch's
    w_tfidf, _ = eng.localize_batch(q, B, sig_list, 10001, incremental=incremental, want_likelihood=False)
    assert np.array_equal(words, w_tfidf)
    want = csr_likelihood(words, sig_list, m)
    assert np.array_equal(bits(like), bits(want))
    assert np.mean(sig_list[np.argmax(like, axis=1)] == places) > 0.5
    # the literal oracle (findPairs on multisets) on a slice
    sw = {int(s): m.sig_words[s - 1] for s in m.sig_ids[:300]}
    for b in (0, 127):
        lit = sim.compute_likelihood(words[b], sig_list[:300], sw)
        assert np.array_equal(bits(like[b, :300]), bits(lit))
    # device entry point and the single-query call give the same bits
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_s = torch.from_numpy(sig_list).cuda()
    d_l = torch.zeros(B * len(sig_list), dtype=torch.float32, device="cuda")
    d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.localize_similarity_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), len(sig_list), 0, d_w.data_ptr(), d_l.data_ptr(), incremental=incremental)
    eng.synchronize()
    assert np.array_equal(d_w.cpu().numpy().reshape(B, F), words)
    assert np.array_equal(bits(d_l.cpu().numpy().reshape(B, -1)), bits(like))
    for b in (3, 64):
        assert np.array_equal(bits(eng.similarity(words[b], sig_list)), bits(like[b]))


def test_word_pairs_on_the_oracle_dictionary_quantisation(c2):
    """The words the similarity batch quantises equal the oracle's (read-only addNewWords), so the word pairs come from the right ids."""
    eng, vocab, ids, m, q, places = c2
    o = orc.OracleDictionary(0, 32, True, 0.8, True)
    o.add_words(ids, vocab)
    o.last_word_id = 49152
    o.update()
    words, like = eng.localize_similarity_batch(q[:2000], 2, m.sig_ids)
    for b in range(2):
        w_o, _ = o.localize_ro(q[b * 1000:(b + 1) * 1000], m.sig_ids, 10001, want_like=False)
        assert np.array_equal(words[b], w_o)


def test_global_descriptors_at_c2_scale_deterministic_and_within_bound(c2):
    import torch

    eng, vocab, ids, m, q, places = c2
    B, F, D = 128, 1000, 4096
    rng = np.random.default_rng(7)
    G = unit(rng, 10000, D)
    eng.gdesc_add(m.sig_ids, G)
    assert eng.gdesc_count() == 10000 and eng.gdesc_dim() == D
    Q = G[places - 1] + 0.3 * unit(rng, B, D)
    Q = (Q / np.linalg.norm(Q, axis=1, keepdims=True)).astype(np.float32)
    sig_list = np.concatenate([EXTRA_IDS, m.sig_ids]).astype(np.int32)
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_g = torch.from_numpy(Q.reshape(-1)).cuda()
    d_s = torch.from_numpy(sig_list).cuda()
    d_l = torch.zeros(B * len(sig_list), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    runs = []
    for _ in range(2):
        eng.localize_similarity_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), len(sig_list), d_g.data_ptr(), 0, d_l.data_ptr())
        eng.synchronize()
        runs.append(d_l.cpu().numpy().reshape(B, -1).copy())
    L = runs[0]
    assert np.array_equal(bits(runs[0]), bits(runs[1]))
    assert np.all(L[:, :2] == 0) and np.all(L[:, 2:4] == 0)  # virtual place, negative id, unknown ids (no descriptor, no words)
    assert_gdesc_close(L[:, 4:], Q, G)
    assert np.all(sig_list[np.argmax(L, axis=1)] == places)
    # the same bits for the same (query, signature) whatever the batch, the position and the entry point
    sel = np.array([127, 5, 77])
    qs = q.reshape(B, F, 32)[sel].reshape(-1, 32)
    words3, L3 = eng.localize_similarity_batch(qs, 3, sig_list, gdesc=Q[sel])
    assert np.array_equal(bits(L3), bits(L[sel]))
    _, L1 = eng.localize_similarity_batch(q.reshape(B, F, 32)[77], 1, sig_list, gdesc=Q[77:78])
    assert np.array_equal(bits(L1[0]), bits(L[77]))
    assert np.array_equal(bits(eng.similarity(words3[0], sig_list, Q[127])), bits(L[127]))
    _, Lhost = eng.localize_similarity_batch(q, B, sig_list, gdesc=Q)
    assert np.array_equal(bits(Lhost), bits(L))
    # mixed presence: signatures without a descriptor fall back to words, and so does every signature for frames without one
    drop = m.sig_ids[::7]
    eng.gdesc_remove(drop)
    words, Lm = eng.localize_similarity_batch(q[:4000], 4, sig_list, gdesc=Q[:4])
    wl = csr_likelihood(words, sig_list, m)
    has = np.isin(sig_list, m.sig_ids) & ~np.isin(sig_list, drop)
    assert np.array_equal(bits(Lm[:, ~has]), bits(wl[:, ~has]))
    assert np.array_equal(bits(Lm[:, has]), bits(L[:4][:, has]))
    _, Ln = eng.localize_similarity_batch(q[:4000], 4, sig_list)
    assert np.array_equal(bits(Ln), bits(wl))
    eng.gdesc_remove(m.sig_ids)
    assert eng.gdesc_count() == 0 and eng.gdesc_dim() == D


# ------------------------------------------------------------------------------------------- index changes --------
def small_world(seed=1, n_words=6000, n_sigs=300, feats=200):
    vocab = synth.make_binary_vocabulary(n_words, 32, seed)
    ids = np.arange(1, n_words + 1, dtype=np.int32)
    m = synth.make_map(ids, n_sigs, feats, seed=seed + 1)
    eng = Engine(max_words=n_words, max_signatures=n_sigs + 10, max_queries=1000, max_batch=8)
    eng.add_words(ids, vocab)
    eng.last_word_id = n_words
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    model = {int(s): list(m.sig_words[s - 1]) for s in m.sig_ids}
    return eng, vocab, ids, m, model


def check_against_model(eng, model, queries, extra=EXTRA_IDS):
    ids = np.concatenate([np.array(sorted(model), np.int32), extra]).astype(np.int32)
    sw = {s: np.asarray(w, np.int64) for s, w in model.items()}
    for qw in queries:
        got = eng.similarity(qw, ids)
        assert np.array_equal(bits(got), bits(word_likelihood([qw], ids, sw)[0]))
    # the invariant: valid(s) equals the references the index holds for s.  A query with one valid word every signature shares has
    # one pair with every signature, so its likelihood is 1 / valid(s).
    refs = {}
    for w in range(1, eng.last_word_id + 1):
        if eng.word_nw(w):
            sg, cn = eng.get_refs(w)
            for s_, c_ in zip(sg.tolist(), cn.tolist()):
                refs[s_] = refs.get(s_, 0) + c_
    shared = eng.last_word_id + 1
    eng.add_words([shared], np.zeros((1, 32), np.uint8))
    eng.last_word_id = shared
    for s in model:
        eng.add_refs(s, [shared])
        model[s].append(shared)
    probe = eng.similarity([shared, -4, 0], list(model))
    for k, s in enumerate(model):
        n = refs.get(s, 0) + 1
        assert n == sum(1 for w in model[s] if w > 0)
        assert probe[k] == np.float32(1) / np.float32(n), (s, probe[k], n)


def test_word_pairs_follow_every_index_change():
    rng = np.random.default_rng(11)
    eng, vocab, ids, m, model = small_world()
    qs = [model[5][:150] + model[5][:20] + [-1, -2, 0], model[9] + [3, 3, 3], [-5, 0], list(rng.integers(1, 6000, 400))]
    check_against_model(eng, model, qs)
    # remove signatures, and words that still have references
    for s in (5, 17, 300):
        eng.remove_sig(s)
        del model[s]
    gone = np.unique(np.concatenate([model[9][:30], model[40][:10]])).astype(np.int32)
    eng.remove_words(gone)
    for s in model:
        model[s] = [w for w in model[s] if w not in set(gone.tolist())]
    eng.update()
    # references added one signature at a time, through add_refs and through quantize with a signature id
    kept = [w for w in range(1, 6001) if w not in set(gone.tolist())]
    eng.add_refs(9, [kept[100], kept[100], kept[2000], -7, 0])
    model[9] += [kept[100], kept[100], kept[2000]]
    frame = synth.flip_bits(vocab[rng.integers(0, 6000, 300)], 0.05, rng)
    w, _ = eng.quantize(frame, 301)
    model[301] = [int(x) for x in w if x > 0]
    check_against_model(eng, model, qs)
    # clear and rebuild
    eng.clear()
    probe = eng.similarity([1, 2, 3], [1, 2, 3])
    assert np.all(probe == 0)
    eng2, vocab2, ids2, m2, model2 = small_world(seed=4, n_sigs=120)
    eng.add_words(ids2, vocab2)
    eng.last_word_id = 6000
    eng.update()
    eng.load_csr(m2.word_ids, m2.row_ptr, m2.sig, m2.cnt)
    check_against_model(eng, {int(s): list(m2.sig_words[s - 1]) for s in m2.sig_ids}, [list(m2.sig_words[3]) + [0, -1]])


def test_word_pairs_after_a_cold_start_equal_incremental_references():
    eng, vocab, ids, m, model = small_world(seed=7, n_sigs=150)
    inc = Engine(max_words=6000, max_signatures=200, max_queries=1000, max_batch=8)
    inc.add_words(ids, vocab)
    inc.last_word_id = 6000
    inc.update()
    for s in m.sig_ids:
        inc.add_refs(int(s), m.sig_words[s - 1])
    q, _ = synth.make_query_frames(vocab, ids, m, 4, 200, seed=9)
    for e in (eng, inc):
        words, like = e.localize_similarity_batch(q, 4, np.concatenate([m.sig_ids, EXTRA_IDS]))
        want = word_likelihood(words, np.concatenate([m.sig_ids, EXTRA_IDS]), {s: np.asarray(w) for s, w in model.items()})
        assert np.array_equal(bits(like), bits(want))


# ------------------------------------------------------------------------------------- global descriptors ---------
@pytest.mark.parametrize("dim", [1, 7, 128, 1000, 4096, 4100])
def test_global_descriptor_values_within_the_bound_of_the_exact_dot(dim):
    rng = np.random.default_rng(dim)
    eng, vocab, ids, m, model = small_world(n_sigs=77, feats=50)
    G = unit(rng, 77, dim)
    if dim == 1:
        G = np.abs(G)  # unit 1-D descriptors are +-1; keep the products >= 0 on this engine
    eng.gdesc_add(m.sig_ids, G)
    Q = unit(rng, 5, dim)
    if dim == 1:
        Q = np.abs(Q)
    q, _ = synth.make_query_frames(vocab, ids, m, 5, 50, seed=1)
    words, like = eng.localize_similarity_batch(q, 5, m.sig_ids, gdesc=Q)  # ns = 77: not a multiple of the 32-signature tile
    for f in range(5):
        for k in range(77):
            exact = sim.exact_dot(Q[f], G[k])
            tol = sim.gdesc_value_tolerance(Q[f], G[k], like[f, k])
            assert abs(float(like[f, k]) - (exact + 1.0) / 2.0) <= tol, (f, k)
        assert np.array_equal(bits(eng.similarity(words[f], m.sig_ids, Q[f])), bits(like[f]))


def test_global_descriptor_store_replace_remove_and_errors():
    import torch

    rng = np.random.default_rng(3)
    eng, vocab, ids, m, model = small_world(n_sigs=40, feats=60)
    G = unit(rng, 40, 8)
    eng.gdesc_add(m.sig_ids[:10], G[:10])
    assert eng.gdesc_count() == 10 and eng.gdesc_dim() == 8
    qg = G[3].copy()
    qw = model[4][:30]
    v = eng.similarity(qw, m.sig_ids[:12], qg)
    assert abs(float(v[3]) - (sim.exact_dot(qg, G[3]) + 1) / 2) <= sim.gdesc_value_tolerance(qg, G[3], v[3])
    wl = word_likelihood([qw], m.sig_ids[:12], {s: np.asarray(w) for s, w in model.items()})[0]
    assert np.array_equal(bits(v[10:]), bits(wl[10:]))  # no descriptor: words
    eng.gdesc_add([4], G[20:21])  # replace
    assert eng.gdesc_count() == 10
    v2 = eng.similarity(qw, m.sig_ids[:12], qg)
    assert abs(float(v2[3]) - (sim.exact_dot(qg, G[20]) + 1) / 2) <= sim.gdesc_value_tolerance(qg, G[20], v2[3])
    eng.gdesc_remove([4, 5, 999])
    assert eng.gdesc_count() == 8
    v3 = eng.similarity(qw, m.sig_ids[:12], qg)
    assert np.array_equal(bits(v3[3:5]), bits(wl[3:5]))
    eng.gdesc_add(m.sig_ids[30:32], G[30:32])  # reuses the two freed rows
    assert eng.gdesc_count() == 10
    v4 = eng.similarity(qw, m.sig_ids[28:34], qg)
    for k, s in enumerate(m.sig_ids[28:34]):
        if s in (31, 32):
            assert abs(float(v4[k]) - (sim.exact_dot(qg, G[s - 1]) + 1) / 2) <= sim.gdesc_value_tolerance(qg, G[s - 1], v4[k])
    assert np.array_equal(bits(eng.similarity(qw, m.sig_ids[:10], qg)[:3]), bits(v[:3]))  # untouched rows keep their values
    with pytest.raises(LcdError) as ex:
        eng.gdesc_add([1], np.ones((1, 9), np.float32))
    assert ex.value.code == -1 and eng.gdesc_dim() == 8
    # a non-normalised pair: the host calls fail like the reference's UASSERT, the device call writes the value
    eng.gdesc_add([1], -np.ones((1, 8), np.float32))
    with pytest.raises(LcdError, match="normalized") as ex:
        eng.similarity(qw, [1, 2], np.ones(8, np.float32))
    assert ex.value.code == -1
    q, _ = synth.make_query_frames(vocab, ids, m, 2, 60, seed=2)
    with pytest.raises(LcdError, match="normalized"):
        eng.localize_similarity_batch(q, 2, [1, 2], gdesc=np.ones((2, 8), np.float32))
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_g = torch.ones(16, dtype=torch.float32, device="cuda")
    d_s = torch.tensor([1, 2], dtype=torch.int32, device="cuda")
    d_l = torch.zeros(4, dtype=torch.float32, device="cuda")
    eng.localize_similarity_batch_dev(d_q.data_ptr(), 2, 60, d_s.data_ptr(), 2, d_g.data_ptr(), 0, d_l.data_ptr())
    eng.synchronize()
    assert float(d_l.cpu()[0]) == np.float32((-8.0 + 1.0) / 2.0)


# ----------------------------------------------------------------------------------------- composition ------------
def test_similarity_calls_leave_tfidf_outputs_unchanged():
    import torch

    rng = np.random.default_rng(5)
    eng, vocab, ids, m, model = small_world(n_sigs=200, feats=150)
    q, _ = synth.make_query_frames(vocab, ids, m, 6, 150, seed=6)
    s = np.concatenate([m.sig_ids, EXTRA_IDS])
    w1, l1 = eng.localize_batch(q, 6, s, 201)
    eng.gdesc_add(m.sig_ids, unit(rng, 200, 64))
    eng.localize_similarity_batch(q, 6, s, gdesc=unit(rng, 6, 64))
    eng.similarity(w1[0], s, unit(rng, 1, 64)[0])
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_s = torch.from_numpy(s.astype(np.int32)).cuda()
    d_l = torch.zeros(6 * len(s), dtype=torch.float32, device="cuda")
    eng.localize_similarity_batch_dev(d_q.data_ptr(), 6, 150, d_s.data_ptr(), len(s), 0, 0, d_l.data_ptr())
    eng.synchronize()
    w2, l2 = eng.localize_batch(q, 6, s, 201)
    assert np.array_equal(w1, w2) and np.array_equal(bits(l1), bits(l2))


def test_similarity_then_verification_of_the_arg_max():
    import torch

    vocab = synth.make_binary_vocabulary(6000, 32, 1)
    ids = np.arange(1, 6001, dtype=np.int32)
    m = synth.make_map(ids, 250, 400, seed=2)
    st = synth.make_signature_store(vocab, ids, m)
    B, F = 5, 400
    q, uv, places, poses = synth.make_query_frames_geo(st, m, B)
    eng = Engine()
    eng.add_words(ids, vocab)
    eng.last_word_id = 6000
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.sig_add_batch(m.sig_ids, st.desc, st.xyz)
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_uv = torch.from_numpy(uv.reshape(-1)).cuda()
    d_s = torch.from_numpy(m.sig_ids).cuda()
    d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
    d_l = torch.zeros(B * 250, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    vp = Engine.verify_params(synth.CAMERA_K4)
    eng.localize_similarity_batch_dev(d_q.data_ptr(), B, F, d_s.data_ptr(), 250, 0, d_w.data_ptr(), d_l.data_ptr())
    eng.verify_top_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, d_l.data_ptr(), d_s.data_ptr(), 250, vp)
    hyp, res = eng.process_fetch(B)
    words = d_w.cpu().numpy().reshape(B, F)
    like = d_l.cpu().numpy().reshape(B, 250)
    want = word_likelihood(words, m.sig_ids, {int(s): m.sig_words[s - 1] for s in m.sig_ids})
    assert np.array_equal(bits(like), bits(want))
    for b in range(B):
        h = int(m.sig_ids[np.argmax(want[b])])
        assert hyp[b] == h == places[b]
        v = orc.verify_pair_cov(st.desc[h - 1], st.xyz[h - 1], q[b * F:(b + 1) * F], uv[b * F:(b + 1) * F], synth.CAMERA_K4)
        r = res[b]
        assert r["ok"] == v["ok"] and r["n_matches"] == len(v["matches"]) and r["n_inliers"] == len(v["inliers"])
        assert np.allclose(r["rvec"], v["rvec"], atol=1e-4) and np.allclose(r["tvec"], v["tvec"], atol=1e-4)
        assert np.allclose(r["covariance"], v["covariance"], rtol=1e-4, atol=1e-9)


def test_sharded_engine_gets_a_state_error():
    eng, vocab, ids, m, model = small_world(n_sigs=20, feats=40)
    eng.shard_set_row_offset(64)
    q, _ = synth.make_query_frames(vocab, ids, m, 1, 40, seed=1)
    calls = [lambda: eng.gdesc_add([1], np.ones((1, 4), np.float32)), lambda: eng.gdesc_remove([1]), lambda: eng.similarity([1, 2], [1]),
             lambda: eng.localize_similarity_batch(q, 1, [1, 2])]
    for c in calls:
        with pytest.raises(LcdError) as ex:
            c()
        assert ex.value.code == -4
