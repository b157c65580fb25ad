"""The TF-IDF likelihood (resolve.cuh score_prep, score.cuh score_kernel<false> + gather_likelihood_kernel) bit for bit against the exact
model of its fixed-point sum (tests/tfidf_model.py), and within the derived bound of the reference's float sum: at the kernel's slice and
walk edges for every LCD_SCORE_BLOCKS, at query, idf and signature edges, at bench scale, through every entry point that produces the
likelihood, and after long edit sequences of the inverted index.  N = 0 gives zeros everywhere (the reference's `if(N)`); N < 0 is
refused."""
import numpy as np
import pytest

import tfidf_model as tm
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import LCD_DESC_F32, LcdError

pytestmark = pytest.mark.gpu

LCD_ERR_INVALID = -1
BLOCKS = [1, 3, 32, 4096]


def assert_bits(got, want, what=""):
    got = np.ascontiguousarray(got, np.float32)
    want = np.ascontiguousarray(want, np.float32)
    assert got.shape == want.shape, what
    diff = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert len(diff) == 0, f"{what}: {len(diff)} values differ, first at {diff[0]}: {got.flat[diff[0]]!r} != {want.flat[diff[0]]!r}"


def assert_oracle_bound(idx, query, sig_ids, n_total, got, self_ref=0):
    o = tm.oracle_likelihood(idx, query, sig_ids, n_total, self_ref)
    ok = tm.within_bound(got, o.like, o.bound)
    assert ok.all(), f"{(~ok).sum()} values outside the bound against the reference's float sum"


def assert_refused(fn):
    with pytest.raises(LcdError) as ex:
        fn()
    assert ex.value.code == LCD_ERR_INVALID and "n_total" in str(ex.value)


def dictionary_engine(n_words, seed=1, **kw):
    eng = Engine(**kw)
    ids = np.arange(1, n_words + 1, dtype=np.int32)
    eng.add_words(ids, synth.make_binary_vocabulary(n_words, 32, seed))
    eng.last_word_id = n_words
    eng.update()
    return eng


def load(eng, idx: tm.Index, words=None):
    """The model's lists into the engine (load_csr), then its ni (set_ni overrides the sums load_csr leaves)."""
    words = sorted(idx.lists) if words is None else words
    rp, sig, cnt = [0], [], []
    for w in words:
        s, c = idx.refs(w)
        sig += s.tolist()
        cnt += c.tolist()
        rp.append(len(sig))
    eng.load_csr(np.array(words, np.int32), np.array(rp, np.int64), np.array(sig, np.int32), np.array(cnt, np.int32))
    nz = np.flatnonzero(np.arange(len(idx.ni)) > 0)
    eng.set_ni(nz, idx.ni[nz])


# ---------------------------------------------------------------- slice and walk edges -----------------------------------------------
S_EDGE = 700          # signatures of the hand-built lists (a list holds a signature once: no list is longer)
N_EDGE = 1000
TOTALS = [0, 1, 255, 256, 257, 511, 513, 767, 769, 4351, 4353, 8191, 8192, 8193, 8447, 8449, 24831, 24833]


def _lengths(total, rng):
    """List lengths summing to `total`, with empty lists first, last, and exactly where a slice of 3 or 32 blocks starts and ends and
    one thread stride (256 postings) after it, and lists ending one posting before and after those points."""
    pts = set()
    for b in (3, 32):
        chunk = -(-total // b) if total else 0
        for k in range(1, b):
            for p in (chunk * k, chunk * k + 256, chunk * k - 1, chunk * k + 1):
                if 0 < p < total:
                    pts.add(p)
    for p in range(256, total, 256):
        pts.add(p)
    pts |= set(int(x) for x in rng.integers(1, max(total, 2), total // 90 + 1) if 0 < x < total)
    cuts = [0] + sorted(pts) + [total]
    # no list longer than S_EDGE
    full = [0]
    for a, b in zip(cuts[:-1], cuts[1:]):
        while b - full[-1] > S_EDGE:
            full.append(full[-1] + S_EDGE)
        full.append(b)
    special = set()
    for b in (3, 32):
        chunk = -(-total // b) if total else 0
        special |= {chunk * k for k in range(1, b)} | {chunk * k + 256 for k in range(1, b)}
    out = [0, 0]   # empty lists first
    for a, b in zip(full[:-1], full[1:]):
        if b > a:
            out.append(b - a)
        if b in special:
            out += [0, 0]   # empty lists exactly at a slice boundary / thread stride: repeated prefix values
    return out + [0, 0]    # and last


@pytest.fixture(scope="module")
def edge_world():
    rng = np.random.default_rng(11)
    lists, cases, w = {}, [], 1
    for total in TOTALS:
        words = []
        for ln in _lengths(total, rng):
            if ln:
                lists[w] = (rng.choice(S_EDGE, ln, replace=False) + 1, rng.integers(1, 4, ln))
            words.append(w)
            w += 1
        assert sum(len(lists[x][0]) for x in words if x in lists) == total and len(words) <= 4096
        cases.append((total, words))
    ni = {s: int(v) for s, v in zip(range(1, S_EDGE + 1), rng.integers(1, 1500, S_EDGE))}
    ni[5] = 1   # ni < nwi for some postings
    return tm.Index(lists, ni), cases, w - 1


@pytest.mark.parametrize("blocks", BLOCKS)
def test_slice_and_walk_edges_for_every_block_count(blocks, edge_world, monkeypatch):
    """Each frame's postings are split into `blocks` slices, each thread binary-searches its first posting and walks forward over the
    repeated prefix values of empty lists.  Every total and every block count gives the model's bits (hence the same bits at every
    setting), and the reference's sum within the bound."""
    monkeypatch.setenv("LCD_SCORE_BLOCKS", str(blocks))
    idx, cases, n_words = edge_world
    eng = dictionary_engine(n_words)
    load(eng, idx)
    sig_ids = np.concatenate([np.arange(1, S_EDGE + 1), [0, -1, S_EDGE + 5, 10 ** 6, 7, 7]]).astype(np.int32)
    rng = np.random.default_rng(blocks)
    for total, words in cases:
        q = np.array(words + list(rng.choice(words, len(words) // 3 + 1)) + [0, -2], np.int32)
        rng.shuffle(q)
        got = eng.score(q, sig_ids, N_EDGE)
        want = tm.gpu_likelihood(idx, q, sig_ids, N_EDGE)
        assert_bits(got, want, f"total {total}, blocks {blocks}")
        assert_oracle_bound(idx, q, sig_ids, N_EDGE, got)
        assert (want != 0).any() == (total > 0)


# ---------------------------------------------------------------- query edges --------------------------------------------------------
@pytest.fixture(scope="module")
def query_world():
    rng = np.random.default_rng(5)
    n_words, S = 6000, 400
    lists = {}
    for w in range(1, n_words + 1):
        k = int(rng.integers(0, 8)) if w % 50 else int(rng.integers(100, S))
        if k:
            lists[w] = (rng.choice(S, k, replace=False) + 1, rng.integers(1, 5, k))
    ni = {s: int(v) for s, v in zip(range(1, S + 1), rng.integers(20, 900, S))}
    return tm.Index(lists, ni), n_words, S


def test_query_edges(query_world):
    idx, n_words, S = query_world
    eng = dictionary_engine(n_words)
    load(eng, idx)
    sig_ids = np.arange(0, S + 3, dtype=np.int32)
    N = S + 1
    rng = np.random.default_rng(6)
    distinct = rng.choice(n_words, 4096, replace=False).astype(np.int32) + 1       # kMaxFrameQueries distinct words
    one = np.full(4096, 50, np.int32)                                                # 4096 copies of one word (a long list)
    nonpos = np.array([0, -1, -5, -(2 ** 31)] * 40, np.int32)                       # only ids <= 0: an all-zero row
    above = np.concatenate([distinct[:300], [10 ** 7, 2 ** 31 - 1, n_words + 1, 65535, 65536, 10 ** 6]]).astype(np.int32)  # ids above the id capacity
    for name, q in (("distinct", distinct), ("one word", one), ("ids <= 0", nonpos), ("above capacity", above)):
        got = eng.score(q, sig_ids, N)
        assert_bits(got, tm.gpu_likelihood(idx, q, sig_ids, N), name)
        assert_oracle_bound(idx, q, sig_ids, N, got)
    assert not eng.score(nonpos, sig_ids, N).any()
    with pytest.raises(LcdError):
        eng.score(np.ones(4097, np.int32), sig_ids, N)
    # removed words take their lists with them
    gone = distinct[:500]
    eng.remove_words(gone)
    idx2 = tm.Index({w: v for w, v in idx.lists.items() if w not in set(gone.tolist())}, dict(enumerate(idx.ni.tolist())))
    got = eng.score(distinct, sig_ids, N)
    assert_bits(got, tm.gpu_likelihood(idx2, distinct, sig_ids, N), "removed words")


def test_batch_of_empty_and_full_frames_equals_each_frame_alone(query_world):
    """lcd_shard_score_ids_dev takes word ids directly: frames with no positive id (nuq = 0) next to frames of thousands of words.  Every
    frame's fixed-point row equals the model's accumulator and the same frame scored alone; N = 0 gives zeros, N < 0 is refused."""
    import torch

    idx, n_words, S = query_world
    eng = dictionary_engine(n_words)
    load(eng, idx)
    rng = np.random.default_rng(8)
    nq = 4096
    frames = np.zeros((6, nq), np.int32)
    frames[1, :3000] = rng.choice(n_words, 3000, replace=False) + 1
    frames[2] = -1
    frames[3] = rng.integers(1, n_words + 1, nq)
    frames[4, 7] = 50
    frames[5, :] = rng.integers(-3, 40, nq)
    sig_ids = np.arange(1, S + 1, dtype=np.int32)
    N = S + 1
    d_sig = torch.from_numpy(sig_ids).cuda()

    def run(rows, n_total):
        d_w = torch.from_numpy(np.ascontiguousarray(rows)).cuda()
        sc = torch.zeros(len(rows) * S, dtype=torch.int64, device="cuda")
        like = torch.zeros(len(rows) * S, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        eng.shard_score_ids_dev(d_w.data_ptr(), len(rows), nq, d_sig.data_ptr(), S, n_total, sc.data_ptr())
        eng.shard_finalize_dev(sc.data_ptr(), len(rows) * S, like.data_ptr())
        eng.synchronize()
        return sc.cpu().numpy().reshape(len(rows), S), like.cpu().numpy().reshape(len(rows), S)

    fixed, like = run(frames, N)
    for b in range(len(frames)):
        acc, amb = tm.gpu_fixed(idx, frames[b], N, self_ref=1)
        assert not amb
        assert np.array_equal(fixed[b], acc[sig_ids]), f"frame {b}"
        assert_bits(like[b], tm.gather(acc, sig_ids), f"frame {b}")
        alone, _ = run(frames[b:b + 1], N)
        assert np.array_equal(alone[0], fixed[b])
    assert not fixed[[0, 2]].any() and fixed[[1, 3, 4]].any(axis=1).all()
    zero, zl = run(frames, 0)
    assert not zero.any() and not zl.any()
    d_w = torch.from_numpy(frames).cuda()
    sc = torch.zeros(len(frames) * S, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    assert_refused(lambda: eng.shard_score_ids_dev(d_w.data_ptr(), len(frames), nq, d_sig.data_ptr(), S, -1, sc.data_ptr()))


# ---------------------------------------------------------------- idf edges ----------------------------------------------------------
SWEEP_NW = list(range(1, 321)) + [511, 512, 999, 1000, 1001, 2047]
SWEEP_N = list(range(1, 61)) + [100, 255, 256, 299, 300, 301, 320, 321, 511, 1000, 1001, 2047, 4096, 10001, 20000, 65536]


def test_idf_sweep_through_single_posting_probes():
    """Word k has nw_k postings: one in a probe signature with nwi = ni = 1 and the rest in filler signatures, so the probe's likelihood
    is idf(N, nw_k) itself (exactly, for |idf| >= 2^-16: the fixed point then loses nothing).  nw == N gives 0 (the word is skipped),
    nw = N - 1 a tiny idf, nw > N a negative one.  The GPU equals the model everywhere and glibc's log10f within two ulps."""
    lists, ni = {}, {}
    probe0 = 3000
    for k, nw in enumerate(SWEEP_NW):
        w = k + 1
        lists[w] = (np.concatenate([[probe0 + k], np.arange(1, nw)]), np.ones(nw, np.int64))
        ni[probe0 + k] = 1
    for s in range(1, max(SWEEP_NW)):
        ni[s] = 7
    idx = tm.Index(lists, ni)
    eng = dictionary_engine(len(SWEEP_NW))
    load(eng, idx)
    words = np.arange(1, len(SWEEP_NW) + 1, dtype=np.int32)
    probes = probe0 + np.arange(len(SWEEP_NW), dtype=np.int32)
    n_diff = n_two = n_all = 0
    for N in SWEEP_N:
        got = eng.score(words, probes, N)
        assert_bits(got, tm.gpu_likelihood(idx, words, probes, N), f"N = {N}")
        idf, amb = tm.idf_gpu(N, SWEEP_NW)
        assert not amb.any()
        big = np.abs(idf) >= 2.0 ** -16
        assert_bits(got[big], idf[big], f"N = {N}: likelihood = idf")
        assert np.all(got[np.array(SWEEP_NW) == N] == 0)
        libm = tm.idf_libm(N, SWEEP_NW)
        d = np.abs(got.astype(np.float64) - libm)
        ulp = np.spacing(np.maximum(np.abs(got), np.abs(libm))).astype(np.float64)
        assert np.all(d[big] <= 2 * ulp[big]), f"N = {N}"
        n_diff += int((got[big] != libm[big]).sum())
        n_two += int((d[big] > ulp[big]).sum())
        n_all += int(big.sum())
        assert_oracle_bound(idx, words, probes, N, got)
    print(f"GPU idf != log10f in {n_diff} of {n_all} (N, nw) pairs, by two ulps in {n_two}")
    assert not eng.score(words, probes, 0).any()                       # N = 0: the reference computes nothing
    assert_refused(lambda: eng.score(words, probes, -1))
    assert_refused(lambda: eng.score(words, probes, -(2 ** 31)))


# ---------------------------------------------------------------- signature edges ----------------------------------------------------
def test_signature_edges():
    eng = dictionary_engine(300, max_signatures=64)
    rng = np.random.default_rng(3)
    refs, ni = {}, {}

    def add(sig, words):
        eng.add_refs(sig, words)
        for w in words:
            if w > 0:
                refs.setdefault(int(w), {}).setdefault(sig, 0)
                refs[int(w)][sig] += 1
        ni[sig] = ni.get(sig, 0) + len(words)

    for s in range(1, 60):
        add(s, rng.integers(1, 301, 40).tolist())
    add(63, [1, 1, 1, 2, 3, 0, -4])
    add(64, [1, 5, 5])                         # the first id past the initial capacity: grows it
    add(50000, [1, 2, 2, 2, 9])                # a much larger one: the new capacity ends right after it
    add(49999, [2, 9, 9])
    q = np.arange(1, 301, dtype=np.int32)
    req = np.array([1, 1, 2, 0, -3, 63, 64, 65, 49999, 50000, 50001, 10 ** 7, 30, 30, 31, 32], np.int32)   # duplicates, <= 0, unknown
    N = 70
    for step in ("grown", "ni = 0", "ni < nwi"):
        if step == "ni = 0":
            eng.set_ni([30, 50000], [0, 0])     # signatures that still have postings
            ni[30] = ni[50000] = 0
        if step == "ni < nwi":
            eng.set_ni([31, 63, 49999], [1, 1, 2])
            ni[31], ni[63], ni[49999] = 1, 1, 2
        idx = tm.Index.from_refs(refs, ni)
        got = eng.score(q, req, N)
        assert_bits(got, tm.gpu_likelihood(idx, q, req, N), step)
        assert_oracle_bound(idx, q, req, N, got)
    assert got[list(req).index(30)] == 0 and got[list(req).index(50000)] == 0 and got[list(req).index(49999)] != 0


# ---------------------------------------------------------------- production scale ---------------------------------------------------
@pytest.mark.parametrize("zipf", [1.0, 1.3])
def test_bench_scale_map(zipf):
    """The bench's shape: 49 152 words, 10 000 signatures of 1000 features; s = 1.3 puts a few words in nearly every signature."""
    ids = np.arange(1, 49153, dtype=np.int32)
    m = synth.make_map(ids, 10000, 1000, seed=2, zipf_s=zipf)
    idx = tm.Index.from_csr(m.word_ids, m.row_ptr, m.sig, m.cnt, m.sig_ids, m.ni)
    eng = dictionary_engine(49152)
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    N = len(m.sig_ids) + 1
    rng = np.random.default_rng(9)
    for k in range(3):
        q = m.sig_words[rng.integers(0, len(m.sig_ids))]
        got = eng.score(q, m.sig_ids, N)
        assert_bits(got, tm.gpu_likelihood(idx, q, m.sig_ids, N), f"query {k}")
        assert_oracle_bound(idx, q, m.sig_ids, N, got)


# ---------------------------------------------------------------- every entry point --------------------------------------------------
def _map_world(n_words=5000, S=300, F=256, f32=False):
    vocab = synth.make_float_vocabulary(n_words, 64, 21) if f32 else synth.make_binary_vocabulary(n_words, 32, 21)
    ids = np.arange(1, n_words + 1, dtype=np.int32)
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=64) if f32 else Engine()
    eng.add_words(ids, vocab)
    eng.last_word_id = n_words
    eng.update()
    m = synth.make_map(ids, S, F, seed=2)
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    return eng, vocab, ids, m, tm.Index.from_csr(m.word_ids, m.row_ptr, m.sig, m.cnt, m.sig_ids, m.ni)


@pytest.mark.parametrize("f32", [False, True], ids=["binary", "float"])
def test_localize_batch(f32):
    eng, vocab, ids, m, idx = _map_world(f32=f32)
    B, F = 5, 256
    if f32:
        rng = np.random.default_rng(4)
        q = np.concatenate([vocab[rng.integers(0, len(ids), F)] + rng.normal(0, 0.02, (F, 64)).astype(np.float32) for _ in range(B)])
    else:
        q, _ = synth.make_query_frames(vocab, ids, m, B, F, seed=4)
    sig_ids = np.concatenate([m.sig_ids, [0, 10 ** 6]]).astype(np.int32)
    N = len(m.sig_ids) + 1
    for incremental in (True, False):
        words, like = eng.localize_batch(q, B, sig_ids, N, incremental=incremental)
        for b in range(B):
            assert_bits(like[b], tm.gpu_likelihood(idx, words[b], sig_ids, N, self_ref=1), f"frame {b}")
            assert_oracle_bound(idx, words[b], sig_ids, N, like[b], self_ref=1)
    _, zero = eng.localize_batch(q, B, sig_ids, 0)
    assert not zero.any()
    assert_refused(lambda: eng.localize_batch(q, B, sig_ids, -1))
    assert_refused(lambda: eng.localize_batch(q, B, sig_ids, -1, want_likelihood=False))
    import torch

    d_q = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    d_sig = torch.from_numpy(sig_ids).cuda()
    d_like = torch.zeros(B * len(sig_ids), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    assert_refused(lambda: eng.localize_batch_dev(d_q.data_ptr(), B, F, d_sig.data_ptr(), len(sig_ids), -1, 0, d_like.data_ptr()))


def test_process_batch():
    vocab = synth.make_binary_vocabulary(6000, 32, 1)
    ids = np.arange(1, 6001, dtype=np.int32)
    m = synth.make_map(ids, 250, 400, seed=2)
    st = synth.make_signature_store(vocab, ids, m)
    B, F = 4, 400
    q, uv, _, _ = synth.make_query_frames_geo(st, m, B)
    eng = Engine()
    eng.add_words(ids, vocab)
    eng.last_word_id = 6000
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.sig_add_batch(m.sig_ids, st.desc, st.xyz)
    idx = tm.Index.from_csr(m.word_ids, m.row_ptr, m.sig, m.cnt, m.sig_ids, m.ni)
    vp = Engine.verify_params(synth.CAMERA_K4)
    N = 251
    words, like, hyp, _ = eng.process_batch(q, uv, B, m.sig_ids, N, vp)
    for b in range(B):
        assert_bits(like[b], tm.gpu_likelihood(idx, words[b], m.sig_ids, N, self_ref=1), f"frame {b}")
    assert like.any(axis=1).all()
    _, zero, _, _ = eng.process_batch(q, uv, B, m.sig_ids, 0, vp)
    assert not zero.any()
    assert_refused(lambda: eng.process_batch(q, uv, B, m.sig_ids, -1, vp))
    import torch

    d_q = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    d_uv = torch.from_numpy(np.ascontiguousarray(uv)).cuda()
    d_sig = torch.from_numpy(m.sig_ids).cuda()
    torch.cuda.synchronize()
    assert_refused(lambda: eng.process_batch_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, d_sig.data_ptr(), len(m.sig_ids), -1, vp))


def test_map_frame():
    """Mapping mode: the frame's own references join the index before the likelihood (self_ref = 0 through lcd_index_score)."""
    rng = np.random.default_rng(3)
    op = Engine.orb_params(synth.CAMERA_K4, n_features=400)
    base = [(synth.make_image(240, 320, 900 + p, bgr=True), synth.make_depth(240, 320, 950 + p)) for p in range(3)]
    frames = [synth.render_view(*base[t % 3], int(rng.integers(-4, 5)), int(rng.integers(-4, 5)), 2.0, rng) for t in range(8)]
    eng = Engine()
    refs, ni = {}, {}
    for t, (img, dep) in enumerate(frames):
        sig = t + 1
        eng.map_detect_async(img, dep, op)
        wm = np.arange(1, sig, dtype=np.int32) if sig > 1 else None
        n_total = 0 if t == len(frames) - 1 else sig
        if t == 4:
            assert_refused(lambda: eng.map_frame(sig, wm, -1))   # refused before the detection is taken: the call can be repeated
        n_kp, words, _, like = eng.map_frame(sig, wm, n_total)
        for w in words:
            if w > 0:
                refs.setdefault(int(w), {}).setdefault(sig, 0)
                refs[int(w)][sig] += 1
        ni[sig] = n_kp
        for w in np.unique(words[words > 0])[::25]:
            s, c = eng.get_refs(int(w))
            assert dict(zip(s.tolist(), c.tolist())) == refs[int(w)]
        if wm is not None:
            idx = tm.Index.from_refs(refs, ni)
            assert_bits(like, tm.gpu_likelihood(idx, words, wm, n_total), f"frame {t}")
            assert_oracle_bound(idx, words, wm, n_total, like)
    assert not like.any() and n_total == 0


@pytest.mark.parametrize("score_parts", [1, 2])
def test_fused_sharded_step_with_one_rank(score_parts, monkeypatch):
    """lcd_shard_process_frames_dev on a one-rank communicator (LCD_SHARD_SCORE_PARTS: the TF-IDF stage whole or in two halves) and
    lcd_process_frames_dev: the likelihood of every frame equals the model fed the word ids the call returned."""
    import torch

    monkeypatch.setenv("LCD_SHARD_SCORE_PARTS", str(score_parts))
    eng = Engine(max_words=8192, max_signatures=400)
    op = Engine.orb_params(synth.CAMERA_K4, n_features=300)
    world = synth.make_place_world(lambda im, dp: eng.orb_detect_describe(im[None], dp[None], op, cap=300)[0], 6, 1500, 120, 300, 240, 320)
    sm = world.smap
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = int(world.word_ids.max())
    eng.update()
    eng.load_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt)
    eng.set_ni(sm.sig_ids, sm.ni)
    eng.sig_add_batch(sm.sig_ids, world.store.desc, world.store.xyz, sm.ni)
    idx = tm.Index.from_csr(sm.word_ids, sm.row_ptr, sm.sig, sm.cnt, sm.sig_ids, sm.ni)
    imgs, deps, _ = synth.make_view_frames(world, 5, seed=4)
    vp = Engine.verify_params(synth.CAMERA_K4, image_size=(320, 240))
    nf, ns = len(imgs), len(sm.sig_ids)
    N = ns + 1
    d_img = torch.from_numpy(imgs).cuda()
    d_dep = torch.from_numpy(deps.view(np.int16)).cuda()
    d_sig = torch.from_numpy(sm.sig_ids).cuda()
    d_rowids = torch.from_numpy(world.word_ids).cuda()
    last = int(world.word_ids.max())
    ext = torch.cuda.ExternalStream(eng.stream)
    out = {}
    with torch.cuda.stream(ext):
        for n_total in (N, 0):
            w0 = torch.zeros(nf * 300, dtype=torch.int32, device="cuda")
            l0 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
            eng.process_frames_dev(d_img.data_ptr(), nf, 320, 240, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, n_total, vp, w0.data_ptr(),
                                   l0.data_ptr(), True, 0.8, True)
            eng.process_fetch(nf)
            out[("plain", n_total)] = (w0.cpu().numpy().reshape(nf, 300), l0.cpu().numpy().reshape(nf, ns))
        assert_refused(lambda: eng.process_frames_dev(d_img.data_ptr(), nf, 320, 240, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, -1, vp))
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        for n_total in (N, 0):
            w1 = torch.zeros(nf * 300, dtype=torch.int32, device="cuda")
            l1 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
            eng.shard_process_frames_dev(d_img.data_ptr(), nf, 320, 240, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, n_total, d_rowids.data_ptr(),
                                         last, vp, w1.data_ptr(), l1.data_ptr(), True, 0.8, True)
            eng.process_fetch(nf)
            out[("shard", n_total)] = (w1.cpu().numpy().reshape(nf, 300), l1.cpu().numpy().reshape(nf, ns))
        l2 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        assert_refused(lambda: eng.shard_process_frames_dev(d_img.data_ptr(), nf, 320, 240, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, -1,
                                                            d_rowids.data_ptr(), last, vp, 0, l2.data_ptr()))
        d_q = torch.zeros(nf * 300 * 32, dtype=torch.uint8, device="cuda")
        assert_refused(lambda: eng.shard_localize_batch_dev(d_q.data_ptr(), nf, 300, d_sig.data_ptr(), ns, -1, d_rowids.data_ptr(), last, 0,
                                                            l2.data_ptr()))
        eng.synchronize()
        eng.shard_comm_destroy()
    for kind in ("plain", "shard"):
        words, like = out[(kind, N)]
        for b in range(nf):
            assert_bits(like[b], tm.gpu_likelihood(idx, words[b], sm.sig_ids, N, self_ref=1), f"{kind} frame {b}")
        assert like.any(axis=1).all()
        assert not out[(kind, 0)][1].any()


# ---------------------------------------------------------------- the index after long edit sequences -------------------------------
class Mirror:
    """The inverted index as the reference keeps it (VisualWord::_references, Memory::getNi) for the edit calls of the C ABI."""

    def __init__(self, words):
        self.refs, self.ni, self.known = {}, {}, set(int(w) for w in words)

    def add_refs(self, sig, words):
        for w in words:
            if w > 0 and w in self.known:
                d = self.refs.setdefault(int(w), {})
                d[sig] = d.get(sig, 0) + 1
        self.ni[sig] = self.ni.get(sig, 0) + len(words)

    def remove_sig(self, sig):
        for d in self.refs.values():
            d.pop(sig, None)
        self.ni[sig] = 0

    def remove_words(self, words):
        for w in words:
            self.refs.pop(int(w), None)
            self.known.discard(int(w))

    def total(self):
        return sum(sum(d.values()) for d in self.refs.values())


def test_index_after_long_edit_sequences():
    rng = np.random.default_rng(17)
    n_words = 400
    eng = dictionary_engine(n_words)
    mir = Mirror(range(1, n_words + 1))
    hot = 200        # one word every signature references: its list is relocated 4 -> 8 -> ... -> 8192 (index_move_kernel)
    touched = set()

    def check(phase):
        for w in sorted(touched):
            s, c = eng.get_refs(w)
            want = sorted(mir.refs.get(w, {}).items())
            assert list(zip(s.tolist(), c.tolist())) == want, f"{phase}: word {w}"
        assert eng.total_refs() == mir.total(), phase
        idx = tm.Index.from_refs(mir.refs, mir.ni)
        q = np.arange(1, n_words + 1, dtype=np.int32)
        sig_ids = np.arange(0, max(mir.ni) + 2, dtype=np.int32)
        N = len([s for s, v in mir.ni.items() if v]) + 1
        assert_bits(eng.score(q, sig_ids, N), tm.gpu_likelihood(idx, q, sig_ids, N), phase)

    # bulk load of the first 100 words, then incremental adds on top of it
    lists = {w: (rng.choice(60, int(rng.integers(1, 30)), replace=False) + 1, rng.integers(1, 3, 30)) for w in range(1, 101)}
    lists = {w: (s, c[:len(s)]) for w, (s, c) in lists.items()}
    rp, sig, cnt = [0], [], []
    for w in range(1, 101):
        sig += lists[w][0].tolist()
        cnt += lists[w][1].tolist()
        rp.append(len(sig))
        for s_, c_ in zip(*lists[w]):
            mir.refs.setdefault(w, {})[int(s_)] = int(c_)
            mir.ni[int(s_)] = mir.ni.get(int(s_), 0) + int(c_)
    eng.load_csr(np.arange(1, 101, dtype=np.int32), np.array(rp, np.int64), np.array(sig, np.int32), np.array(cnt, np.int32))
    touched |= set(range(1, 101))
    check("load_csr")
    for s in range(1, 8300):   # many small calls with repeated words
        words = [hot] * int(rng.integers(1, 3)) + rng.integers(1, 120, int(rng.integers(0, 4))).tolist() + [0]
        eng.add_refs(s, words)
        mir.add_refs(s, words)
        touched |= {w for w in words if w > 0}
    assert eng.word_nw(hot) == 8299
    check("adds")
    removed = rng.choice(np.arange(1, 8300), 700, replace=False)
    for s in removed:
        eng.remove_sig(int(s))
        mir.remove_sig(int(s))
    check("remove_sig")
    for s in removed[:300]:
        words = [hot, int(rng.integers(1, 120)), int(rng.integers(1, 120))]
        eng.add_refs(int(s), words)
        mir.add_refs(int(s), words)
    check("re-add")
    gone = [3, 50, 101, 119]
    eng.remove_words(gone)
    mir.remove_words(gone)
    for s in range(8300, 8400):
        words = [hot, 3, 50, int(rng.integers(1, 120))]      # removed words: skipped, but counted in ni
        eng.add_refs(s, words)
        mir.add_refs(s, words)
    check("remove_words")
    sel = rng.choice(np.arange(1, 8400), 200, replace=False)
    vals = rng.integers(0, 5, 200)
    eng.set_ni(sel, vals)
    for s, v in zip(sel, vals):
        mir.ni[int(s)] = int(v)
    check("set_ni")
