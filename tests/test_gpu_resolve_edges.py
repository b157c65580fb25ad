"""The new-word loop (resolve_rounds in resolve.cuh, resolve_rounds_l2 in l2_path.cuh) at its edges, through every caller, against
the CPU oracle's sequential VWDictionary::addNewWords / findNN / localisation and RegistrationVis matching: alternating chains that
need all 32 passes of a chunk (on chunk starts and across the chunk boundaries), ties in the multimap's insertion order, NNDR products
at the float boundary, frames of 1 to 4096 descriptors, the quantiser's modes, both 2-NN kernels that feed the loop, the two-shard
emulation and pair matching.  Cases: resolve_cases.py; that they reach their edge on the oracle: test_oracle_resolve_cases.py.

Bar: identical word ids, new-word count, last word id, not-indexed size and signature references; then findNN on the created
descriptors and knn2 after update() bit-identical (the created words reached the not-indexed tail in creation order)."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, sharding, synth
from rtabmap_b200.capi import LCD_DESC_F32
import resolve_cases as rc
from test_gpu_parity import assert_likelihood_close

pytestmark = pytest.mark.gpu

K4 = synth.CAMERA_K4


def pair(words, float_desc=False, nndr=0.8, cmp_new=True, incremental=True):
    """An engine and an oracle holding `words` as ids 1..n, indexed."""
    dim = words.shape[1]
    eng = Engine(desc_type=LCD_DESC_F32 if float_desc else 0, desc_dim=dim, max_queries=rc.MAX_FRAME)
    o = orc.OracleDictionary(int(float_desc), dim, incremental, nndr, cmp_new)
    if len(words):
        ids = np.arange(1, len(words) + 1, dtype=np.int32)
        eng.add_words(ids, words)
        o.add_words(ids, words)
    eng.last_word_id = len(words)
    o.last_word_id = len(words)
    eng.update()
    o.update()
    return eng, o


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


def quantize_both(eng, o, frame, sig=7, incremental=True, nndr=0.8, cmp_new=True, tag=""):
    """lcd_dict_quantize against addNewWords, then every check of the module docstring; returns the oracle's word ids."""
    prev = o.last_word_id
    o.set_params(incremental, nndr, cmp_new)
    g, n_new = eng.quantize(frame, sig, incremental, nndr, cmp_new)
    w = o.add_new_words(frame, sig)
    assert np.array_equal(g, w), (tag, np.flatnonzero(g != w)[:10])
    assert n_new == o.last_word_id - prev, tag
    assert eng.last_word_id == o.last_word_id and eng.not_indexed_size() == o.not_indexed_size() == n_new, tag
    for wid in np.unique(w):
        s1, c1 = eng.get_refs(int(wid))
        s2, c2 = o.get_refs(int(wid))
        assert np.array_equal(s1, s2) and np.array_equal(c1, c2), (tag, int(wid))
    first = np.unique(w, return_index=True)[1]
    created = frame[first[w[first] > prev]]
    if len(created):
        assert np.array_equal(eng.find_nn(created, incremental, nndr), o.find_nn(created)), tag
    eng.update()
    o.update()
    probe = np.concatenate([frame[:64], created[:64]])
    for a, b in zip(eng.knn2(probe), o.knn2(probe)):
        assert same(a, b), tag
    return w


# ---------------------------------------------------------------------------------------------------------------- 1. chains
@pytest.mark.parametrize("lead", rc.LEADS)
@pytest.mark.parametrize("length,dim,kernel", [(50, 16, None), (100, 32, 0), (100, 32, 1), (200, 64, None)])
def test_binary_chain(length, dim, kernel, lead):
    """A chain alternating over its whole length: in an aligned chunk lane k changes at pass k, so a pass loop stopped early leaves
    lanes wrong.  32-byte descriptors under both 2-NN kernels (XOR/POPC 0, tensor cores 1)."""
    chain, index = rc.binary_chain(length, dim, seed=length)
    eng, o = pair(index)
    if kernel is not None:
        eng.nn_select(kernel)
    w = quantize_both(eng, o, rc.chain_frame(chain, lead, seed=lead), tag=(length, dim, lead))
    if kernel is not None:
        assert eng.nn_last_kernel == kernel
    assert rc.alternation(w, lead, length, len(index))


@pytest.mark.parametrize("lead", rc.LEADS)
@pytest.mark.parametrize("length,dim", rc.F32_CHAINS)
def test_float_chain_exact_kernel(length, dim, lead):
    chain, index = rc.float_chain(length, dim, seed=length)
    eng, o = pair(index, float_desc=True)
    eng.nn_select(0)
    w = quantize_both(eng, o, rc.chain_frame(chain, lead, seed=lead), tag=(length, dim, lead))
    assert eng.nn_last_kernel == 0
    assert rc.alternation(w, lead, length, len(index))


@pytest.mark.parametrize("length,dim", rc.F32_CHAINS)
def test_float_chain_tensor_filter(length, dim):
    """The dictionary padded with far words to 4096 rows, so the fp16 tensor-core filter + exact re-rank feeds the loop."""
    chain, index = rc.float_chain(length, dim, seed=length)
    pad = rc.far_rows(4096 - len(index), dim, np.float32, np.random.default_rng(dim))
    words = np.concatenate([index, pad])
    for lead in rc.LEADS:
        eng, o = pair(words, float_desc=True)
        eng.nn_select(1)
        w = quantize_both(eng, o, rc.chain_frame(chain, lead, seed=lead), tag=(length, dim, lead))
        assert eng.nn_last_kernel == 1, "the tensor-core filter did not run"
        assert rc.alternation(w, lead, length, len(index))


@pytest.mark.parametrize("cmp_new,incremental", [(False, True), (True, False)])
def test_binary_chain_modes(cmp_new, incremental):
    """Kp/NewWordsComparedTogether=false (warp0_compact: every chain row creates a word) and a fixed dictionary (nearest word)."""
    chain, index = rc.binary_chain(100, 32, seed=100)
    eng, o = pair(index, cmp_new=cmp_new, incremental=incremental)
    for lead in rc.LEADS:
        w = quantize_both(eng, o, rc.chain_frame(chain, lead, seed=lead), incremental=incremental, cmp_new=cmp_new, tag=lead)
        if not incremental:
            assert (w > 0).all() and (w <= len(index)).all()
        else:
            assert len(np.unique(w[lead:lead + 100])) == 100


@pytest.mark.parametrize("cmp_new", [True, False])
def test_float_chain_modes(cmp_new):
    chain, index = rc.float_chain(100, 128, seed=100)
    eng, o = pair(index, float_desc=True, cmp_new=cmp_new, incremental=cmp_new)
    for lead in rc.LEADS:
        quantize_both(eng, o, rc.chain_frame(chain, lead, seed=lead), incremental=cmp_new, cmp_new=cmp_new, tag=lead)


# ---------------------------------------------------------------------------------------------------------------- 2. ties
def test_tie_index_word_wins_over_new_word():
    d, f = rc.tie_index_vs_new(32, seed=1)
    eng, o = pair(d)
    w = quantize_both(eng, o, f)
    assert w[0] == 2 and (w[[1, 31, 32, 33, 64, 95]] == 1).all()


def test_tie_earlier_new_word_wins_and_one_entry_rule():
    eng, o = pair(np.zeros((0, 32), np.uint8))
    w = quantize_both(eng, o, rc.tie_new_vs_new(32, seed=2))
    assert w[0] == 1 and w[1] == 2 and (w[list(rc.TIE_COPIES)] == 1).all()


def test_tie_lower_index_row_wins():
    d, f = rc.tie_index_pair(32, seed=3)
    eng, o = pair(d)
    w = quantize_both(eng, o, f)
    assert (w[[0, 31, 32, 63]] == 4).all()


def test_find_nn_indexed_word_wins_over_not_indexed_word():
    """findNN searches the index and the not-indexed words: an indexed and a not-indexed row at distance 0, the indexed row wins."""
    rng = np.random.default_rng(8)
    d = rc.far_rows(600, 32, np.uint8, rng)
    eng, o = pair(d)
    extra = rc.far_rows(40, 32, np.uint8, rng)
    extra[7] = d[5]
    extra[30] = d[450]
    ids = np.arange(601, 641, dtype=np.int32)
    eng.add_words(ids, extra)
    o.add_words(ids, extra)
    q = np.concatenate([d[[5, 450]], extra[[7, 30]], rc.far_rows(60, 32, np.uint8, rng)])
    got = eng.find_nn(q, True, 0.8)
    assert np.array_equal(got, o.find_nn(q))
    assert list(got[:4]) == [6, 451, 6, 451]


# ---------------------------------------------------------------------------------------------------------------- 3. NNDR boundary
@pytest.mark.parametrize("gap", [1, 40])
@pytest.mark.parametrize("via", ["index", "new"])
@pytest.mark.parametrize("nndr,best,second,accept", rc.NNDR_CASES)
def test_nndr_boundary(nndr, best, second, accept, via, gap):
    """best > nndr * second in float: (8, 10) and (7, 10) at 0.7 accept, (9, 11) rejects, with the second-best an index word or a
    word this frame created in the same chunk (gap 1) or an earlier one (gap 40)."""
    d, f, q, row = rc.nndr_case(best, second, via, 32, seed=best * 100 + second, gap=gap)
    eng, o = pair(d, nndr=nndr)
    w = quantize_both(eng, o, f, nndr=nndr)
    assert (w[q] == row + 1) == accept
    eng2, o2 = pair(d, nndr=nndr)   # findNN takes the same decision
    assert np.array_equal(eng2.find_nn(f, True, nndr), o2.find_nn(f))


# ---------------------------------------------------------------------------------------------------------------- 4. frame sizes
@pytest.mark.parametrize("n", rc.FRAME_SIZES)
def test_frame_sizes(n):
    rng = np.random.default_rng(n)
    vocab = rng.integers(0, 256, (2000, 32), dtype=np.uint8)
    eng, o = pair(vocab)
    quantize_both(eng, o, rc.mixed_frame(vocab, n, seed=1000 + n), tag=n)


def test_full_frame_into_an_empty_dictionary():
    """4096 random descriptors: every one is new, phase A of the last chunk scans 4064 earlier words."""
    eng, o = pair(np.zeros((0, 32), np.uint8))
    w = quantize_both(eng, o, rc.far_rows(rc.MAX_FRAME, 32, np.uint8, np.random.default_rng(9)))
    assert o.last_word_id == rc.MAX_FRAME and np.array_equal(w, np.arange(1, rc.MAX_FRAME + 1))


def test_repeated_descriptors_shuffled():
    eng, o = pair(np.zeros((0, 32), np.uint8))
    quantize_both(eng, o, rc.repeated_frame(32, seed=4))


@pytest.mark.parametrize("float_desc", [False, True])
def test_chain_at_the_end_of_a_full_frame(float_desc):
    chain, index = rc.float_chain(100, 128, seed=5) if float_desc else rc.binary_chain(100, 32, seed=5)
    eng, o = pair(index, float_desc=float_desc)
    lead = rc.MAX_FRAME - 100
    w = quantize_both(eng, o, rc.chain_frame(chain, lead, seed=6, total=rc.MAX_FRAME))
    assert rc.alternation(w, lead, 100, len(index))


# ---------------------------------------------------------------------------------------------------------------- 5. callers
def chain_world(n_pad=3000, n_sig=200, feats=150):
    """32-byte chain of 100 with its index words, the dictionary padded with far words, and a map over it."""
    chain, index = rc.binary_chain(100, 32, seed=100)
    words = np.concatenate([index, rc.far_rows(n_pad, 32, np.uint8, np.random.default_rng(11))])
    ids = np.arange(1, len(words) + 1, dtype=np.int32)
    m = synth.make_map(ids, n_sig, feats, seed=2)
    return chain, words, ids, m


def chain_batch(chain, words, B, F, chain_at):
    """B frames of F rows: near copies of dictionary words, and at batch positions chain_at the chain at lead 0 or 29."""
    rng = np.random.default_rng(12)
    q = np.stack([rc.mixed_frame(words, F, seed=20 + b) for b in range(B)])
    for k, b in enumerate(chain_at):
        lead = rc.LEADS[k % 2]
        q[b, lead:lead + len(chain)] = chain
    return q


def test_quantize_with_signature_refs():
    chain, words, ids, m = chain_world()
    eng, o = pair(words)
    for t, lead in enumerate(rc.LEADS, start=1):
        quantize_both(eng, o, rc.chain_frame(chain, lead, seed=lead), sig=100 + t)
        assert eng.total_refs() == o.total_refs()


def test_localize_batch_chain_frames():
    chain, words, ids, m = chain_world()
    eng, o = pair(words)
    for d in (eng, o):
        d.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    B, F = 6, 160
    q = chain_batch(chain, words, B, F, chain_at=(0, 3, 5))
    got_w, got_l = eng.localize_batch(q.reshape(B * F, 32), B, m.sig_ids, len(m.sig_ids) + 1)
    for b in range(B):
        w_o, l_o = o.localize_ro(q[b], m.sig_ids, len(m.sig_ids) + 1)
        assert np.array_equal(got_w[b], w_o), f"frame {b}"
        assert_likelihood_close(got_l[b], l_o)
    for b, lead in ((0, 0), (3, 29)):
        assert rc.alternation(got_w[b], lead, len(chain), len(words))
    assert eng.not_indexed_size() == 0


@pytest.mark.parametrize("by_frame", [False, True])
def test_two_word_range_shards_on_chain_frames(by_frame):
    """The two-shard emulation of test_gpu_shard.py (collectives as torch ops on one device) on chain frames."""
    import torch

    chain, words, ids, m = chain_world()
    W, S, B, F = len(words), len(m.sig_ids), 4, 160
    q = chain_batch(chain, words, B, F, chain_at=(1, 2))
    full, o = pair(words)
    for d in (full, o):
        d.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    full.set_ni(m.sig_ids, m.ni)
    want_w, want_l = full.localize_batch(q.reshape(B * F, 32), B, m.sig_ids, S + 1)
    for b in range(B):
        assert np.array_equal(want_w[b], o.localize_ro(q[b], m.sig_ids, S + 1)[0])
    last = W
    G = 2
    shards = []
    for r in range(G):
        r0, r1 = sharding.shard_rows(W, G, r)
        e = Engine()
        e.add_words(ids[r0:r1], words[r0:r1])
        e.last_word_id = last
        e.update()
        e.shard_set_row_offset(r0)
        e.load_csr(*sharding.shard_csr(m.word_ids, m.row_ptr, m.sig, m.cnt, ids[r0:r1]))
        e.set_ni(m.sig_ids, m.ni)
        shards.append(e)
    nq = B * F
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_rowids = torch.from_numpy(ids).cuda()
    d_sig = torch.from_numpy(m.sig_ids.astype(np.int32)).cuda()
    d_nv = torch.from_numpy(np.full(B, F, np.int32)).cuda()
    torch.cuda.synchronize()
    keys = []
    for e in shards:
        k = torch.zeros(nq * 2, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        e.shard_knn2_keys_dev(d_q.data_ptr(), nq, k.data_ptr())
        e.synchronize()
        keys.append(k)
    keys_all = torch.cat(keys)
    scores = []
    if not by_frame:
        words_out = []
        for e in shards:
            w_ = torch.zeros(nq, dtype=torch.int32, device="cuda")
            sc = torch.zeros(B * S, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            e.shard_resolve_score_dev(d_q.data_ptr(), B, F, keys_all.data_ptr(), G, d_rowids.data_ptr(), W, last, d_sig.data_ptr(), S, S + 1,
                                      w_.data_ptr(), sc.data_ptr())
            e.synchronize()
            words_out.append(w_)
            scores.append(sc)
        assert torch.equal(words_out[0], words_out[1])
        words_all = words_out[0]
    else:
        parts = []
        for r, e in enumerate(shards):
            f0, f1 = sharding.shard_rows(B, G, r)
            w_ = torch.zeros((f1 - f0) * F, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            e.shard_resolve_frames_dev(d_q.data_ptr(), f0, f1 - f0, B, F, keys_all.data_ptr(), G, d_rowids.data_ptr(), last, d_nv.data_ptr(),
                                       w_.data_ptr())
            e.synchronize()
            parts.append(w_)
        words_all = torch.cat(parts)
        for e in shards:
            sc = torch.zeros(B * S, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            e.shard_score_ids_dev(words_all.data_ptr(), B, F, d_sig.data_ptr(), S, S + 1, sc.data_ptr())
            e.synchronize()
            scores.append(sc)
    total = scores[0] + scores[1]
    like = torch.zeros(B * S, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    shards[0].shard_finalize_dev(total.data_ptr(), B * S, like.data_ptr())
    shards[0].synchronize()
    got_w = words_all.cpu().numpy().reshape(B, F)
    got_l = like.cpu().numpy().reshape(B, S)
    for b in range(B):
        assert np.array_equal(got_w[b], want_w[b]), f"frame {b}"
        assert np.allclose(got_l[b], want_l[b], rtol=1e-6, atol=1e-7), f"frame {b}"
    assert rc.alternation(got_w[1], 0, len(chain), W) and rc.alternation(got_w[2], 29, len(chain), W)


# ---------------------------------------------------------------------------------------------------------------- 7. pair matching
def binary_pair_sets(length, dim):
    """FROM: the planted neighbours, then the chain (the chain alternates in the FROM dictionary); TO: the chain reversed, copies of
    every fourth planted neighbour (words seen once on each side: correspondences) and random rows."""
    chain, index = rc.binary_chain(length, dim, seed=length)
    to = np.concatenate([chain[::-1], index[::4], rc.far_rows(length // 2, dim, np.uint8, np.random.default_rng(dim))])
    return np.concatenate([index, chain]), to


@pytest.mark.parametrize("length,dim", rc.BIN_CHAINS)
def test_binary_pair_matching(length, dim):
    src, to = binary_pair_sets(length, dim)
    eng = Engine(desc_dim=dim)
    cap = max(len(src), len(to))
    F = np.zeros((2, cap, dim), np.uint8)
    T = np.zeros((2, cap, dim), np.uint8)
    F[0, :len(src)], T[0, :len(to)] = src, to
    F[1, :len(to)], T[1, :len(src)] = to, src   # and the other way round
    fid, tid = eng.match_pairs(F, T, [len(src), len(to)], [len(to), len(src)])
    for i, (a, b) in enumerate(((src, to), (to, src))):
        f_o, t_o = orc.match_pair(a, b)
        assert np.array_equal(fid[i, :len(a)], f_o) and np.array_equal(tid[i, :len(b)], t_o), i
    assert rc.alternation(fid[0], len(src) - length, length, int(fid[0, :len(src) - length].max()))


def random_geometry(rng, n_from, n_to):
    xyz = np.stack([rng.uniform(-2, 2, n_from), rng.uniform(-1.5, 1.5, n_from), rng.uniform(1, 5, n_from)], 1).astype(np.float32)
    uv = np.stack([rng.uniform(0, 640, n_to), rng.uniform(0, 480, n_to)], 1).astype(np.float32)
    return xyz, uv


@pytest.mark.parametrize("length,dim", rc.F32_CHAINS)
def test_float_pair_matching(length, dim):
    """lcd_verify_batch's correspondences on float chains (FROM: the chain, which alternates from its second row on; TO: the chain
    reversed and far rows) against the oracle's verification."""
    chain, _ = rc.float_chain(length, dim, seed=length)
    rng = np.random.default_rng(dim)
    to = np.concatenate([chain[::-1], rc.far_rows(length // 2, dim, np.float32, rng)])
    xyz, uv = random_geometry(rng, len(chain), len(to))
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=dim)
    cap = len(to)
    F = np.zeros((1, cap, dim), np.float32)
    X = np.full((1, cap, 3), np.nan, np.float32)
    F[0, :len(chain)], X[0, :len(chain)] = chain, xyz
    g = eng.verify_batch(F, X, to[None], uv[None], K4, [len(chain)], [len(to)])[0]
    v = orc.verify_pair_cov(chain, xyz, to, uv, K4)
    assert np.array_equal(g["matches"], v["matches"]) and g["ok"] == v["ok"]
    assert len(v["matches"]) > 0


def test_cached_from_dictionary_equals_the_uncached_call():
    """A stored signature holding the chain set: the fused call builds its FROM dictionary, then reads it from the cache; both equal
    lcd_verify_batch on the same pair."""
    import torch

    src, to = binary_pair_sets(100, 32)
    rng = np.random.default_rng(3)
    xyz, uv = random_geometry(rng, len(src), len(to))
    eng = Engine(desc_dim=32)
    pad = len(src) - len(to)
    g = eng.verify_batch(src[None], xyz[None], np.concatenate([to, np.zeros((pad, 32), np.uint8)])[None],
                         np.concatenate([uv, np.zeros((pad, 2), np.float32)])[None], K4, [len(src)], [len(to)])[0]
    v = orc.verify_pair_cov(src, xyz, to, uv, K4)
    assert np.array_equal(g["matches"], v["matches"]) and len(v["matches"]) > 0
    eng.sig_add_batch([5], src[None], xyz[None])
    d_q = torch.from_numpy(to.reshape(-1)).cuda()
    d_uv = torch.from_numpy(uv.reshape(-1)).cuda()
    d_l = torch.ones(1, dtype=torch.float32, device="cuda")
    d_s = torch.tensor([5], dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for _ in range(2):   # the first call builds the cached dictionary, the second reads it
        eng.verify_top_dev(d_q.data_ptr(), d_uv.data_ptr(), 1, len(to), d_l.data_ptr(), d_s.data_ptr(), 1, Engine.verify_params(K4))
        hyp, res = eng.process_fetch(1)
        assert list(hyp) == [5]
        assert res[0]["n_matches"] == len(g["matches"]) and res[0]["ok"] == g["ok"] and res[0]["n_inliers"] == len(g["inliers"])
