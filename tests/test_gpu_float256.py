"""256-D float descriptors (SuperPoint's unit-length rows) through every float-engine call, against the dimension-generic oracle.

The 2-NN at 256-D runs on kernels of its own shape: the fp16 filter streams each 256-word tile as four 32 KB K slices
(nn_tensor_f32.cuh), and the exact kernels read the query a 64-float chunk at a time (l2_path.cuh).  The cases sit at the edges of
that tiling: the exact / filter crossover (4096 rows), the 256-row word tiles and the 16-tile bound pre-pass.  The verification,
decision and sharding tests of the 64-D and 128-D engines are re-run here at 256-D through their own helpers."""
import types

import numpy as np
import pytest

import test_gpu_decide_f32 as df
import test_gpu_shard_f32 as sf
import test_gpu_verify_f32 as vf
from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import LCD_DESC_F32
from test_gpu_boundary import _cv2_cross, _cv2_knn
from test_gpu_float import float_vocab, noisy

pytestmark = pytest.mark.gpu

D = 256


def pair(n_words, seed=1, incremental=True, nndr=0.8, cmp_new=True, vocab=None):
    vocab = float_vocab(n_words, D, seed) if vocab is None else vocab
    ids = np.arange(1, n_words + 1, dtype=np.int32) * 2
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=D)
    o = orc.OracleDictionary(1, D, incremental, nndr, cmp_new)
    if n_words:
        eng.add_words(ids, vocab)
        o.add_words(ids, vocab)
    last = int(ids.max()) if n_words else 0
    eng.last_word_id = last
    o.last_word_id = last
    eng.update()
    o.update()
    return eng, o, vocab, ids


def same_bits(g, w):
    assert np.array_equal(g[0], w[0]) and np.array_equal(g[2], w[2])
    assert np.array_equal(g[1].view(np.uint32), w[1].view(np.uint32)) and np.array_equal(g[3].view(np.uint32), w[3].view(np.uint32))


def queries(vocab, n, rng, seed=99):
    q = float_vocab(n, D, seed)
    if len(vocab) >= 8:
        k = min(n // 3, len(vocab))
        q[:k] = noisy(vocab[rng.integers(0, len(vocab), k)], 0.05, rng)
        q[k] = vocab[len(vocab) // 2]
    return q


# --------------------------------------------------------------------------------------------------------------------- 2-NN
@pytest.mark.parametrize("n_words", [0, 1, 2, 700, 4095, 4096, 4097, 8193])
def test_knn2_bit_exact(n_words):
    """Exact kernel below 4096 rows, filter from 4096 on (4097 and 8193: a one-row last tile)."""
    eng, o, vocab, ids = pair(n_words, seed=n_words + 5)
    rng = np.random.default_rng(7)
    q = queries(vocab, 300, rng)
    g = eng.knn2(q)
    assert eng.nn_last_kernel == (1 if n_words >= 4096 else 0)
    same_bits(g, o.knn2(q))
    if n_words >= 4096:
        eng.nn_select(0)
        same_bits(eng.knn2(q), g)


@pytest.mark.parametrize("n_words", [2000, 9000])
def test_duplicates_across_tile_and_prepass_edges_resolve_to_the_lowest_row(n_words):
    """Copies of one row at both sides of the 32-row exact tiles, the 256-row word tiles, the 128-row fallback tiles and the end of
    the 16-tile bound pre-pass (row 4096): the nearest is the lowest copy, the second the next one, in every kernel."""
    vocab = float_vocab(n_words, D, 3)
    copies = [r for r in (31, 32, 127, 128, 255, 256, 4095, 4096, 8191) if r < n_words]
    vocab[copies] = vocab[copies[-1]]
    eng, o, _, ids = pair(n_words, vocab=vocab)
    q = np.concatenate([vocab[copies[-1]][None], noisy(vocab[copies[-1]][None], 1e-3, np.random.default_rng(1))])
    for sel in (1, 0):
        eng.nn_select(sel)
        g = eng.knn2(q)
        same_bits(g, o.knn2(q))
        assert g[0][0] == ids[copies[0]] and g[2][0] == ids[copies[1]]


@pytest.mark.parametrize("n_words", [9000, 70001])
def test_filter_is_bit_identical_to_the_exact_kernel_with_near_ties_at_eps(n_words):
    """Rows planted so that their squared distance exceeds the nearest one's by 0.5 ... 2 times the filter's margin 2 eps
    (eps ~ 2.24e-3 for unit rows at 256-D): the candidate lists cut right through them, and the result must not change."""
    vocab = float_vocab(n_words, D, 3 * n_words)
    rng = np.random.default_rng(17)
    base = rng.integers(0, n_words - 64, 40)
    eps = (1.02 * 2.0 ** -9 + 2.0 ** -13) + 2.0 ** -14 * 2 + 4e-6
    for j, b in enumerate(base):
        u = rng.standard_normal(D).astype(np.float32)
        u -= (u @ vocab[b]) * vocab[b]
        u /= np.linalg.norm(u)
        d1 = 0.01 + 0.002 * (j % 5)
        for k, f in enumerate((0.5, 0.95, 1.0, 1.05, 2.0)):
            t = np.sqrt(d1 + f * 2 * eps)
            vocab[b + 1 + k] = vocab[b] + np.float32(t) * u
        vocab[b + 6] = vocab[b] + np.float32(np.sqrt(d1)) * u
    eng, o, _, ids = pair(n_words, vocab=vocab)
    q = float_vocab(700, D, 5)
    q[:40] = vocab[base]
    q[40:300] = noisy(vocab[rng.integers(0, n_words, 260)], 0.05, rng)
    q[300:330] = vocab[rng.integers(0, n_words, 30)]
    q[330] = 0.0
    q[331:340] *= 30.0
    eng.nn_select(1)
    g = eng.knn2(q)
    assert eng.nn_last_kernel == 1
    n_fb, n_cand, _ = eng.nn_f32_stats(len(q))
    assert n_cand >= 2 * len(q) - 2
    eng.nn_select(0)
    x = eng.knn2(q)
    assert eng.nn_last_kernel == 0
    same_bits(g, x)
    same_bits((g[0][:100], g[1][:100], g[2][:100], g[3][:100]), o.knn2(q[:100]))


def test_overflowing_lists_and_out_of_range_values_fall_back_to_the_exact_scan():
    n_words = 12000
    vocab = float_vocab(n_words, D, 31)
    vocab[2000:2400] = vocab[7]
    vocab[5000:5200] = vocab[8] * np.float32(1.0 + 1e-4)
    eng, o, _, ids = pair(n_words, vocab=vocab)
    rng = np.random.default_rng(32)
    q = noisy(vocab[rng.integers(0, n_words, 64)], 0.03, rng)
    q[0] = vocab[7]
    q[1] = noisy(vocab[7:8], 0.01, rng)[0]
    q[2] = vocab[8]
    q[3] = 1.0e6
    q[4, 5] = np.float32(7.0e4)
    eng.nn_select(1)
    g = eng.knn2(q)
    assert eng.nn_last_kernel == 1
    n_fb, _, _ = eng.nn_f32_stats(len(q))
    assert n_fb >= 4
    eng.nn_select(0)
    same_bits(g, eng.knn2(q))
    same_bits(g, o.knn2(q))
    assert g[0][0] == ids[7] and g[2][0] == ids[2000]
    big = float_vocab(1, D, 33) * np.float32(1.0e7)
    eng.nn_select(1)
    eng.add_words([2 * n_words + 2], big)
    eng.update()
    g2 = eng.knn2(q)
    assert eng.nn_last_kernel == 0
    eng.nn_select(0)
    same_bits(g2, eng.knn2(q))


def test_cached_word_image_follows_add_remove_and_update():
    eng, o, vocab, ids = pair(6000, seed=77)
    rng = np.random.default_rng(78)
    for t in range(1, 6):
        frame = np.concatenate([noisy(vocab[rng.integers(0, 6000, 150)], 0.04, rng), float_vocab(60, D, 1000 + t)])
        frame[200:205] = frame[195:200] + np.float32(1e-3)
        eng.update()
        o.update()
        g, n_new = eng.quantize(frame, t)
        w = o.add_new_words(frame, t)
        assert eng.nn_last_kernel == 1
        assert np.array_equal(g, w), f"frame {t}"
        if t == 3:
            victims = np.asarray(ids[100:140])
            eng.remove_words(victims)
            o.remove_words(victims)
    q = noisy(vocab[rng.integers(0, 6000, 50)], 0.05, rng)
    q[:10] = frame[150:160]
    assert np.array_equal(eng.find_nn(q, True, 0.8), o.find_nn(q))
    same_bits(eng.knn2(q), o.knn2(q))
    eng.update()
    o.update()
    assert np.array_equal(eng.find_nn(q, True, 0.8), o.find_nn(q))
    same_bits(eng.knn2(q), o.knn2(q))


# ------------------------------------------------------------------------------------------------------------- quantiser
@pytest.mark.parametrize("n_words", [1500, 6000])
@pytest.mark.parametrize("cmp_new", [True, False])
def test_incremental_stream(n_words, cmp_new):
    eng, o, vocab, ids = pair(n_words, seed=11, cmp_new=cmp_new)
    rng = np.random.default_rng(13)
    for t in range(1, 5):
        f = float_vocab(160, D, 100 + t)
        f[:60] = noisy(vocab[rng.integers(0, n_words, 60)], 0.03, rng)
        f[100:130] = noisy(f[60:90], 0.02, rng)
        prev_last = o.last_word_id
        got, n_new = eng.quantize(f, t, cmp_new=cmp_new)
        want = o.add_new_words(f, t)
        assert np.array_equal(got, want), f"frame {t}"
        assert n_new == len(np.unique(want[want > prev_last])) and n_new > 0
        assert eng.last_word_id == o.last_word_id and eng.not_indexed_size() == o.not_indexed_size()
        eng.update()
        o.update()
        assert eng.indexed_size() == o.indexed_size()
    probe = noisy(vocab[rng.integers(0, n_words, 50)], 0.04, rng)
    assert np.array_equal(eng.find_nn(probe), o.find_nn(probe))


@pytest.mark.parametrize("incremental", [True, False])
def test_localize_batch_matches_oracle_at_any_batch_position(incremental):
    n_words = 5000
    eng, o, vocab, ids = pair(n_words, seed=21, incremental=incremental)
    m = synth.make_map(ids, 200, 150, seed=2)
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    o.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    rng = np.random.default_rng(5)
    B, F = 4, 150
    frames = [noisy(vocab[rng.integers(0, n_words, F)], 0.05, rng) for _ in range(B)]
    frames[1][100:] = float_vocab(50, D, 40)
    words, like = eng.localize_batch(np.concatenate(frames), B, m.sig_ids, 201, incremental=incremental)
    for b in range(B):
        w_o, l_o = o.localize(frames[b], 9999, m.sig_ids, 201)
        assert np.array_equal(words[b], w_o), f"frame {b}"
        assert np.allclose(like[b], l_o, atol=1e-4, rtol=1e-4)
    order = [2, 0, 3, 1]
    w2, l2 = eng.localize_batch(np.concatenate([frames[i] for i in order]), B, m.sig_ids, 201, incremental=incremental)
    for k, i in enumerate(order):
        assert np.array_equal(w2[k], words[i]) and np.array_equal(l2[k].view(np.uint32), like[i].view(np.uint32))


# ---------------------------------------------------------------------------------------------------------- verification
def test_verify_batch_matches_oracle():
    vf.test_verify_batch_matches_oracle(D)


def test_verify_ties_and_duplicates_match_oracle():
    vf.test_ties_and_duplicates_match_oracle(D)


@pytest.mark.parametrize("cap", [1, 128, 129, 4096])
def test_verify_caps(cap):
    rng = np.random.default_rng(600 + cap)
    eng = vf.float_engine(D)
    for which in range(4):
        assert eng.verify_static_smem(which) >= 0
    counts = [(cap, cap), (max(cap - 1, 0), cap), (cap, 1), (0, cap)] + ([(1000, 1000)] if cap >= 1000 else [])
    scenes = [vf.make_scene(rng, nf, nt, D) for nf, nt in counts]
    g = vf.batch(eng, [(s[0], s[1]) for s in scenes], [(s[2], s[3]) for s in scenes], cap, D)
    for b, s in enumerate(scenes):
        vf.assert_oracle(g[b], vf.oracle(*s[:4]), (cap, counts[b]))
    eng.close()


def test_fused_query_equals_verify_batch():
    vf.test_fused_query_equals_verify_batch_through_the_store_life_cycle(D)


def test_process_batch_equals_localize_then_verify():
    vf.test_process_batch_equals_localize_then_verify(D)


def test_verify_same_bits_at_any_batch_position():
    vf.test_same_bits_at_any_batch_position_and_call(D)


def test_match_bf_against_cv2():
    import cv2

    rng = np.random.default_rng(9)
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=D)
    cap = 400
    T = rng.normal(0, 1, (3, cap, D)).astype(np.float32)
    T /= np.linalg.norm(T, axis=2, keepdims=True)
    Q = (T[:, rng.permutation(cap)] + rng.normal(0, 0.05, T.shape)).astype(np.float32)
    T[2, 40] = T[2, 3]                       # duplicates across the 32-row tiles: ties go to the lowest index
    T[2, 33] = T[2, 3]
    nq, nt = [400, 123, 400], [380, 400, 65]
    i1, d1, i2, d2 = eng.match_bf(Q, T, nq, nt)
    c1, cd, _, _ = eng.match_bf(Q, T, nq, nt, cross_check=True)
    for i in range(3):
        o1, od1, o2, od2 = _cv2_knn(Q[i, :nq[i]], T[i, :nt[i]], cv2.NORM_L2SQR)
        assert np.array_equal(i1[i, :nq[i]], o1) and np.array_equal(i2[i, :nq[i]], o2)
        assert np.allclose(d1[i, :nq[i]], od1, rtol=1e-5) and np.allclose(d2[i, :nq[i]], od2, rtol=1e-5)
        oc, _ = _cv2_cross(Q[i, :nq[i]], T[i, :nt[i]], cv2.NORM_L2SQR)
        assert np.array_equal(c1[i, :nq[i]], oc)


# ------------------------------------------------------------------------------------------------ decision and sharding
@pytest.fixture(scope="module")
def fworld256():
    return df.fworld.__wrapped__(types.SimpleNamespace(param=D))  # the 64 / 128-D world, built at 256-D


def test_localize_decide_verify_decided(fworld256):
    df.test_localize_decide_verify_decided(fworld256)


@pytest.mark.parametrize("incremental", [True, False])
@pytest.mark.parametrize("by_frame", [False, True])
@pytest.mark.parametrize("G", [2, 3, 4])
def test_word_range_shards_equal_one_engine(G, by_frame, incremental):
    sf.test_float_word_range_shards_equal_one_engine(G, D, by_frame, incremental)


def test_fused_localize_with_a_single_rank_communicator_equals_the_unsharded_call():
    import torch

    vocab, ids, m, q, _ = sf._world(2, D)
    eng = sf._float_engine(D, ids, vocab, m, int(ids.max()))
    q = np.ascontiguousarray(q[[0, 2, 3, 4, 5]])
    F = sf.F
    nf, ns, last = q.shape[0], len(m.sig_ids), int(ids.max())
    ext = torch.cuda.ExternalStream(eng.stream)
    with torch.cuda.stream(ext):
        d_q = torch.from_numpy(q.reshape(-1)).cuda()
        d_sig = torch.from_numpy(m.sig_ids).cuda()
        d_rowids = torch.from_numpy(ids).cuda()
        w0 = torch.zeros(nf * F, dtype=torch.int32, device="cuda")
        l0 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        eng.localize_batch_dev(d_q.data_ptr(), nf, F, d_sig.data_ptr(), ns, ns + 1, w0.data_ptr(), l0.data_ptr())
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        try:
            w1 = torch.full((nf * F,), -7, dtype=torch.int32, device="cuda")
            l1 = torch.full((nf * ns,), -1.0, dtype=torch.float32, device="cuda")
            for _ in range(2):
                eng.shard_localize_batch_dev(d_q.data_ptr(), nf, F, d_sig.data_ptr(), ns, ns + 1, d_rowids.data_ptr(), last, w1.data_ptr(),
                                             l1.data_ptr())
            eng.synchronize()
            assert torch.equal(w0, w1) and torch.equal(l0, l1)
        finally:
            eng.shard_comm_destroy()
    assert (w0.cpu().numpy() > last).any() and (l0.cpu().numpy() > 0).any()
