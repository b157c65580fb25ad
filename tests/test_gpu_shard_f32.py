"""Word-range sharding of FLOAT-descriptor dictionaries through the C ABI.

1. Emulated shards on ONE GPU (all-gather = concatenation, all-reduce = sum), as tests/test_gpu_shard.py does for binary descriptors:
   G float engines each own a range of the rows and their posting lists; both stage-2 variants must reproduce one unsharded engine —
   word ids bit for bit, and the likelihood bit for bit too, since the scores are exact fixed-point sums whose order cannot matter.
   The workload plants the cases where the float search changes kernel per shard: a shard below the fp16 filter's row minimum (exact
   CUDA-core kernel) next to shards above it, a row beyond fp16 range in one shard only (that shard alone leaves the filter), queries
   that overflow the candidate list on one shard (exact fallback), NNDR rejects and near-duplicate new descriptors inside a frame.
2. C4 size: 1.1 M rows over 4 shards against the reference's own rtflann answer and the oracle's new-word pass.
3. lcd_shard_localize_batch_dev on a communicator of one rank equals lcd_localize_batch_dev on the same engine, float and binary."""
import numpy as np
import pytest

from golden_util import ref_knn2
from oracle import oracle_py as orc
from rtabmap_b200 import Engine, LcdError, sharding, synth

pytestmark = pytest.mark.gpu

LCD_DESC_F32 = 1
LCD_ERR_CAPACITY, LCD_ERR_STATE = -3, -4
TF_MIN_ROWS = 4096                       # nn_tensor_f32.cuh kTfMinRows: smaller dictionaries use the exact kernel
S, F, B = 300, 256, 7
SMALL, LARGE = 3000, 5000                # rows of shard 0 (exact kernel) and of every other shard (fp16 filter)
BLOCK_SRC, BLOCK = SMALL + 100, slice(SMALL + 500, SMALL + 920)   # 420 copies of one row of shard 1: its neighbours overflow the lists


def _bounds(G):
    edges = np.cumsum([0, SMALL] + [LARGE] * (G - 1))
    return [(int(a), int(b)) for a, b in zip(edges[:-1], edges[1:])]


def _world(G, dim):
    W = SMALL + LARGE * (G - 1)
    vocab = synth.make_float_vocabulary(W, dim, 21 + G)
    vocab[BLOCK] = vocab[BLOCK_SRC]
    if G >= 3:
        vocab[W - 10, 0] = np.float32(7.0e4)   # beyond fp16 range: the last shard stays on the exact kernel
    ids = np.arange(1, W + 1, dtype=np.int32) * 2
    m = synth.make_map(ids, S, F, seed=2)
    rng = np.random.default_rng(5 + G)
    id2row = np.full(int(ids.max()) + 1, -1, np.int64)
    id2row[ids] = np.arange(W)
    q = np.empty((B, F, dim), np.float32)
    for f in range(B):
        rows = id2row[m.sig_words[rng.integers(0, S), rng.permutation(F)]]
        d = vocab[rows] + rng.normal(0, 0.02, (F, dim)).astype(np.float32)
        perm = rng.permutation(F)
        new, ovf = perm[:F // 5], perm[F // 5:F // 5 + 8]
        d[new] = synth.make_float_vocabulary(len(new), dim, 1000 + 10 * G + f)       # unrelated: NNDR rejects, new words
        d[new[1::4]] = d[new[0::4]][:len(new[1::4])] + np.float32(1e-3)            # near copies of new descriptors in the frame
        d[ovf] = vocab[BLOCK_SRC] + rng.normal(0, 0.02, (len(ovf), dim)).astype(np.float32)
        q[f] = d
    q[1, 200:] = 0                              # a short frame: 200 valid descriptors, zero padding rows
    n_valid = np.full(B, F, np.int32)
    n_valid[1] = 200
    return vocab, ids, m, np.ascontiguousarray(q), n_valid


def _float_engine(dim, ids, vocab, m, last, r0=0):
    e = Engine(desc_type=LCD_DESC_F32, desc_dim=dim)
    e.add_words(ids, vocab)
    e.last_word_id = last
    e.update()
    if r0:
        e.shard_set_row_offset(r0)
    e.load_csr(*sharding.shard_csr(m.word_ids, m.row_ptr, m.sig, m.cnt, ids))
    e.set_ni(m.sig_ids, m.ni)
    return e


@pytest.mark.parametrize("incremental", [True, False])
@pytest.mark.parametrize("by_frame", [False, True])
@pytest.mark.parametrize("dim", [64, 128])
@pytest.mark.parametrize("G", [2, 3, 4])
def test_float_word_range_shards_equal_one_engine(G, dim, by_frame, incremental):
    import torch

    vocab, ids, m, q, n_valid = _world(G, dim)
    last = int(ids.max())
    full = _float_engine(dim, ids, vocab, m, last)
    want_w, want_l = [], []
    for b in range(B):   # per-frame calls: the reference for the short frame is the frame with only its valid descriptors
        w_, l_ = full.localize_batch(q[b, :n_valid[b]], 1, m.sig_ids, S + 1, incremental)
        want_w.append(w_[0])
        want_l.append(l_[0])

    bounds = _bounds(G)
    shards = [_float_engine(dim, ids[r0:r1], vocab[r0:r1], m, last, r0) for r0, r1 in bounds]
    nq = B * F
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_rowids = torch.from_numpy(ids).cuda()
    d_sig = torch.from_numpy(m.sig_ids.astype(np.int32)).cuda()
    d_nv = torch.from_numpy(n_valid).cuda()
    torch.cuda.synchronize()
    keys = []
    for r, e in enumerate(shards):
        k = torch.zeros(nq * 2, dtype=torch.int64, device="cuda")     # two u64 keys per query
        torch.cuda.synchronize()
        e.shard_knn2_keys_dev(d_q.data_ptr(), nq, k.data_ptr())
        e.synchronize()
        big = G >= 3 and r == G - 1
        assert e.nn_last_kernel == (0 if r == 0 or big else 1), f"shard {r}: rows {bounds[r]}"
        if r == 1:
            assert e.nn_f32_stats(nq)[0] > 0, "no query overflowed its candidate list on shard 1"
        keys.append(k)
    assert bounds[0][1] - bounds[0][0] < TF_MIN_ROWS <= bounds[1][1] - bounds[1][0]
    keys_all = torch.cat(keys)          # "all-gather"
    scores = []
    if not by_frame:
        words = []
        for e in shards:
            w_ = torch.zeros(nq, dtype=torch.int32, device="cuda")
            sc = torch.zeros(B * S, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            e.shard_resolve_score_dev(d_q.data_ptr(), B, F, keys_all.data_ptr(), G, d_rowids.data_ptr(), len(ids), last, d_sig.data_ptr(), S,
                                      S + 1, w_.data_ptr(), sc.data_ptr(), incremental)
            e.synchronize()
            words.append(w_)
            scores.append(sc)
        assert all(torch.equal(words[0], w_) for w_ in words[1:])      # the replicated pass is deterministic
        words_all = words[0]
    else:
        parts = []
        for r, e in enumerate(shards):
            f0, f1 = sharding.shard_rows(B, G, r)      # uneven: 7 frames over 2, 3 or 4 ranks
            w_ = torch.zeros((f1 - f0) * F, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            e.shard_resolve_frames_dev(d_q.data_ptr(), f0, f1 - f0, B, F, keys_all.data_ptr(), G, d_rowids.data_ptr(), last, d_nv.data_ptr(),
                                       w_.data_ptr(), incremental)
            e.synchronize()
            parts.append(w_)
        words_all = torch.cat(parts)    # "all-gather" of the word ids
        for e in shards:
            sc = torch.zeros(B * S, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            e.shard_score_ids_dev(words_all.data_ptr(), B, F, d_sig.data_ptr(), S, S + 1, sc.data_ptr())
            e.synchronize()
            scores.append(sc)
    total = torch.stack(scores).sum(0)  # "all-reduce(sum)"
    like = torch.zeros(B * S, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    shards[0].shard_finalize_dev(total.data_ptr(), B * S, like.data_ptr())
    shards[0].synchronize()
    got_w = words_all.cpu().numpy().reshape(B, F)
    got_l = like.cpu().numpy().reshape(B, S)
    n_new = 0
    for b in range(B):
        if by_frame or n_valid[b] == F:   # the replicated variant has no per-frame counts: the short frame is the by-frame variant's job
            assert np.array_equal(got_w[b, :n_valid[b]], want_w[b]), f"frame {b}"
            assert np.array_equal(got_l[b], want_l[b]), f"frame {b}"
            n_new += int((want_w[b] > last).sum())
        if by_frame:
            assert not got_w[b, n_valid[b]:].any()
    assert (n_new > 0) == incremental     # new words exist exactly in the incremental mode


def test_c4_float_quantiser_over_four_word_range_shards():
    """The inputs of test_gpu_configs.py::test_c4_float_quantiser_over_a_million_rows (1.1 M rows of 64-D, the same 96 queries) over four
    shards: the merged keys give rtflann's ids and distances bit for bit, and the resolve of the merged keys the oracle's word ids."""
    import torch

    W = 1_100_000
    vocab = synth.make_float_vocabulary(W, 64, 21)
    ids = np.arange(1, W + 1, dtype=np.int32)
    rng = np.random.default_rng(22)
    nq = 96
    src = rng.integers(0, W, nq)
    src[:8] = np.array([0, 1, W - 1, W - 2, 1 << 20, (1 << 20) - 1, (1 << 20) + 1, 524288])
    q = vocab[src] + rng.normal(0, 0.02, (nq, 64)).astype(np.float32)
    q[-16:] = synth.make_float_vocabulary(16, 64, 99)
    q[-8:-4] = q[-16:-12] + np.float32(1e-3)
    q = np.ascontiguousarray(q, np.float32)

    G = 4
    d_q = torch.from_numpy(q).cuda()
    keys = []
    shards = []
    for r in range(G):
        r0, r1 = sharding.shard_rows(W, G, r)
        e = Engine(desc_type=LCD_DESC_F32, desc_dim=64, max_words=r1 - r0 + 4096)
        e.add_words(ids[r0:r1], vocab[r0:r1])
        e.last_word_id = W
        e.update()
        e.shard_set_row_offset(r0)
        k = torch.zeros(nq * 2, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        e.shard_knn2_keys_dev(d_q.data_ptr(), nq, k.data_ptr())
        e.synchronize()
        assert e.nn_last_kernel == 1
        keys.append(k)
        shards.append(e)
    keys_all = torch.cat(keys)
    merged = sharding.merge_top2(keys_all.cpu().numpy().view(np.uint64).reshape(G, nq, 2))
    rows = (merged & np.uint64(0xFFFFFFFF)).astype(np.int64)
    dist = (merged >> np.uint64(32)).astype(np.uint32).view(np.float32)
    r_idx, r_dist = ref_knn2(vocab, q)
    assert np.array_equal(rows, r_idx) and np.array_equal(dist, r_dist)
    # word ids: resolve of the gathered keys on one rank, against VWDictionary::addNewWords of the unsharded oracle
    d_rowids = torch.from_numpy(ids).cuda()
    w_ = torch.zeros(nq, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    shards[0].shard_resolve_frames_dev(d_q.data_ptr(), 0, 1, 1, nq, keys_all.data_ptr(), G, d_rowids.data_ptr(), W, 0, w_.data_ptr())
    shards[0].synchronize()
    o = orc.OracleDictionary(1, 64, True, 0.8, True)
    o.add_words(ids, vocab)
    o.last_word_id = W
    o.update()
    w = o.add_new_words(q, 7)
    g = w_.cpu().numpy()
    assert np.array_equal(g, w) and (g > W).sum() >= 8


def _binary_setup():
    W = 6000
    vocab = synth.make_binary_vocabulary(W, 32, 21)
    ids = np.arange(1, W + 1, dtype=np.int32) * 2
    m = synth.make_map(ids, S, F, seed=2)
    q, _ = synth.make_query_frames(vocab, ids, m, 5, F, seed=5)
    e = Engine()
    e.add_words(ids, vocab)
    e.last_word_id = int(ids.max())
    e.update()
    e.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    e.set_ni(m.sig_ids, m.ni)
    return e, ids, m, np.ascontiguousarray(q).reshape(5, F, 32)


def _float_setup():
    vocab, ids, m, q, _ = _world(2, 64)
    e = _float_engine(64, ids, vocab, m, int(ids.max()))
    return e, ids, m, np.ascontiguousarray(q[[0, 2, 3, 4, 5]])   # five full frames


@pytest.mark.parametrize("kind", ["float64", "binary32"])
def test_fused_localize_with_a_single_rank_communicator_equals_the_unsharded_call(kind, monkeypatch):
    """lcd_shard_localize_batch_dev on a communicator of ONE rank: every collective degenerates to a copy, the two-half search pipeline
    (5 frames: halves of 3 and 2) and the exchange bookkeeping still run, and the result must equal lcd_localize_batch_dev."""
    import torch

    eng, ids, m, q = _float_setup() if kind == "float64" else _binary_setup()
    nf, ns = q.shape[0], len(m.sig_ids)
    last = int(ids.max())
    ext = torch.cuda.ExternalStream(eng.stream)
    with torch.cuda.stream(ext):
        d_q = torch.from_numpy(q.reshape(-1)).cuda()
        d_sig = torch.from_numpy(m.sig_ids).cuda()
        d_rowids = torch.from_numpy(ids).cuda()
        w0 = torch.zeros(nf * F, dtype=torch.int32, device="cuda")
        l0 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        with pytest.raises(LcdError) as err:          # no communicator yet
            eng.shard_localize_batch_dev(d_q.data_ptr(), nf, F, d_sig.data_ptr(), ns, ns + 1, d_rowids.data_ptr(), last, w0.data_ptr(), l0.data_ptr())
        assert err.value.code == LCD_ERR_STATE
        eng.localize_batch_dev(d_q.data_ptr(), nf, F, d_sig.data_ptr(), ns, ns + 1, w0.data_ptr(), l0.data_ptr())
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        try:
            with pytest.raises(LcdError) as err:
                eng.shard_localize_batch_dev(d_q.data_ptr(), 1, 4097, d_sig.data_ptr(), ns, ns + 1, d_rowids.data_ptr(), last, w0.data_ptr(),
                                             l0.data_ptr())
            assert err.value.code == LCD_ERR_CAPACITY
            for parts in ("1", "2"):
                monkeypatch.setenv("LCD_SHARD_SCORE_PARTS", parts)
                w1 = torch.full((nf * F,), -7, dtype=torch.int32, device="cuda")
                l1 = torch.full((nf * ns,), -1.0, dtype=torch.float32, device="cuda")
                for _ in range(2):  # twice: the exchange buffers and events are reused
                    eng.shard_localize_batch_dev(d_q.data_ptr(), nf, F, d_sig.data_ptr(), ns, ns + 1, d_rowids.data_ptr(), last, w1.data_ptr(),
                                                 l1.data_ptr())
                eng.synchronize()
                assert torch.equal(w0, w1), f"word ids, LCD_SHARD_SCORE_PARTS={parts}"
                assert torch.equal(l0, l1), f"likelihood, LCD_SHARD_SCORE_PARTS={parts}"
        finally:
            eng.shard_comm_destroy()
    assert (w0.cpu().numpy() > last).any() and (l0.cpu().numpy() > 0).any()
