"""Float descriptors (LCD_DESC_F32: SURF-64 / SURF-128 / SIFT sized rows) through the C ABI against the oracle, whose squared-L2
2-NN is pinned to the reference's own compiled rtflann (tests/test_oracle_ref.py).  Bar: identical neighbours, bit-identical
distances, identical word ids for the incremental / fixed quantiser and findNN, likelihood within 1e-4."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import LCD_DESC_F32

pytestmark = pytest.mark.gpu


def float_vocab(n, dim, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, dim)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)          # SURF / SIFT descriptors are unit length
    return v.astype(np.float32)


def pair(n_words, dim, seed=1, incremental=True, nndr=0.8):
    vocab = float_vocab(n_words, dim, seed)
    ids = np.arange(1, n_words + 1, dtype=np.int32) * 2
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=dim)
    o = orc.OracleDictionary(1, dim, incremental, nndr, True)
    if n_words:
        eng.add_words(ids, vocab)
        o.add_words(ids, vocab)
    last = int(ids.max()) if n_words else 0
    eng.last_word_id = last
    o.last_word_id = last
    eng.update()
    o.update()
    return eng, o, vocab, ids


def noisy(rows, sigma, rng):
    q = rows + sigma * rng.standard_normal(rows.shape).astype(np.float32)
    return (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("dim,n_words", [(64, 0), (64, 1), (64, 2), (64, 700), (64, 5000), (128, 900)])
def test_knn2_float_bit_exact(dim, n_words):
    eng, o, vocab, ids = pair(n_words, dim, seed=dim + n_words)
    rng = np.random.default_rng(7)
    q = float_vocab(300, dim, 99)
    if n_words >= 700:
        q[:100] = noisy(vocab[rng.integers(0, n_words, 100)], 0.05, rng)
        q[100] = vocab[5]
        q[101] = vocab[5]
    g = eng.knn2(q)
    w = o.knn2(q)
    assert np.array_equal(g[0], w[0]) and np.array_equal(g[2], w[2])
    assert np.array_equal(g[1].view(np.uint32), w[1].view(np.uint32)) and np.array_equal(g[3].view(np.uint32), w[3].view(np.uint32))


def test_knn2_float_ties_resolve_to_lowest_row():
    vocab = float_vocab(500, 64, 3)
    vocab[77] = vocab[9]
    vocab[300] = vocab[9]
    ids = np.arange(1, 501, dtype=np.int32)
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=64)
    eng.add_words(ids, vocab)
    eng.update()
    id1, d1, id2, d2 = eng.knn2(vocab[9:10])
    assert (id1[0], d1[0], id2[0], d2[0]) == (10, 0.0, 78, 0.0)


@pytest.mark.parametrize("dim", [64, 128])
def test_incremental_stream_float(dim):
    """Mapping mode: frames quantised one after the other with update() in between; words created inside a frame are compared
    together (Kp/NewWordsComparedTogether) — ids, number of new words and the index must follow the oracle frame by frame."""
    eng, o, vocab, ids = pair(1500, dim, seed=11)
    rng = np.random.default_rng(13)
    for t in range(1, 6):
        f = float_vocab(160, dim, 100 + t)
        f[:60] = noisy(vocab[rng.integers(0, 1500, 60)], 0.03, rng)      # revisits of known words
        f[100:130] = noisy(f[60:90], 0.02, rng)                         # near-duplicates inside the frame
        prev_last = o.last_word_id
        got, n_new = eng.quantize(f, t)
        want = o.add_new_words(f, t)
        assert np.array_equal(got, want), f"frame {t}"
        assert n_new == len(np.unique(want[want > prev_last])) and n_new > 0
        assert eng.last_word_id == o.last_word_id and eng.not_indexed_size() == o.not_indexed_size()
        eng.update()
        o.update()
        assert eng.indexed_size() == o.indexed_size()
    probe = noisy(vocab[rng.integers(0, 1500, 50)], 0.04, rng)
    assert np.array_equal(eng.find_nn(probe), o.find_nn(probe))


def test_fixed_dictionary_and_localize_float():
    eng, o, vocab, ids = pair(3000, 64, seed=21, incremental=False)
    m = synth.make_map(ids, 200, 150, seed=2)
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    o.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    rng = np.random.default_rng(5)
    B, F = 3, 150
    q = np.concatenate([noisy(vocab[rng.integers(0, 3000, F)], 0.05, rng) for _ in range(B)])
    words, like = eng.localize_batch(q, B, m.sig_ids, 201, incremental=False)
    for b in range(B):
        w_o, l_o = o.localize(q[b * F:(b + 1) * F], 9999, m.sig_ids, 201)
        assert np.array_equal(words[b], w_o), f"frame {b}"
        assert np.allclose(like[b], l_o, atol=1e-4, rtol=1e-4)


def test_float_engine_rejects_binary_only_calls():
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=64)
    with pytest.raises(Exception):
        eng.match_pairs(np.zeros((1, 8, 64), np.float32), np.zeros((1, 8, 64), np.float32), [8], [8])


# ---------------------------------------------------------------- tensor-core filter + exact re-rank (nn_tensor_f32.cuh) ----------
@pytest.mark.parametrize("dim,n_words", [(64, 4096), (64, 20000), (64, 70001), (128, 9000)])
def test_tensor_filter_is_bit_identical_to_the_exact_kernel(dim, n_words):
    """Dictionaries of >= 4096 float rows go through the wgmma fp16 GEMM filter + exact re-rank; ids and fp32 distances must equal
    the exact CUDA-core scan (and the rtflann-pinned oracle) bit for bit."""
    eng, o, vocab, ids = pair(n_words, dim, seed=3 * dim + n_words)
    rng = np.random.default_rng(17)
    q = float_vocab(700, dim, 5)
    q[:300] = noisy(vocab[rng.integers(0, n_words, 300)], 0.05, rng)
    q[300:330] = vocab[rng.integers(0, n_words, 30)]          # exact copies: distance 0
    q[330] = 0.0                                              # zero vector
    q[331:340] *= 30.0                                        # long vectors: large distances, large error bound
    eng.nn_select(1)
    g = eng.knn2(q)
    assert eng.nn_last_kernel == 1, "the tensor-core filter did not run"
    eng.nn_select(0)
    x = eng.knn2(q)
    assert eng.nn_last_kernel == 0
    for a, b in zip(g, x):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    w = o.knn2(q[:200])
    assert np.array_equal(g[0][:200], w[0]) and np.array_equal(g[2][:200], w[2])
    assert np.array_equal(g[1][:200].view(np.uint32), w[1].view(np.uint32)) and np.array_equal(g[3][:200].view(np.uint32), w[3].view(np.uint32))


def test_tensor_filter_overflowing_lists_and_out_of_range_values_fall_back_to_the_exact_scan():
    dim, n_words = 64, 12000
    vocab = float_vocab(n_words, dim, 31)
    vocab[2000:2400] = vocab[7]                 # 401 identical rows: every one of them ties for nearest -> the list overflows
    vocab[5000:5200] = vocab[8] * np.float32(1.0 + 1e-4)  # 200 rows within the error bound of each other
    ids = np.arange(1, n_words + 1, dtype=np.int32)
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=dim)
    eng.add_words(ids, vocab)
    eng.last_word_id = n_words
    eng.update()
    rng = np.random.default_rng(32)
    q = noisy(vocab[rng.integers(0, n_words, 64)], 0.03, rng)
    q[0] = vocab[7]
    q[1] = noisy(vocab[7:8], 0.01, rng)[0]
    q[2] = vocab[8]
    q[3] = 1.0e6                                 # does not fit fp16: exact scan for this query
    q[4, 5] = np.float32(7.0e4)
    eng.nn_select(1)
    g = eng.knn2(q)
    assert eng.nn_last_kernel == 1
    eng.nn_select(0)
    x = eng.knn2(q)
    for a, b in zip(g, x):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert g[0][0] == 8 and g[2][0] == 2001      # ties resolve to the lowest rows: row 7 (id 8), then row 2000 (id 2001)
    # a dictionary row outside the fp16 range: noticed while its image is built, the engine stays on the exact kernel
    big = float_vocab(1, dim, 33) * np.float32(1.0e7)
    eng.nn_select(1)
    eng.add_words([n_words + 1], big)
    eng.update()
    g2 = eng.knn2(q)
    assert eng.nn_last_kernel == 0
    eng.nn_select(0)
    x2 = eng.knn2(q)
    for a, b in zip(g2, x2):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_tensor_filter_incremental_stream_matches_oracle():
    """Mapping mode on a float dictionary large enough for the tensor path: new words join the cached fp16 image row by row."""
    eng, o, vocab, ids = pair(6000, 64, seed=77)
    rng = np.random.default_rng(78)
    for t in range(1, 7):
        frame = np.concatenate([noisy(vocab[rng.integers(0, 6000, 150)], 0.04, rng), float_vocab(60, 64, 1000 + t)])
        frame[200:205] = frame[195:200] + np.float32(1e-3)   # near copies of descriptors that become new words in this frame
        eng.update()
        o.update()
        g, n_new = eng.quantize(frame, t)
        w = o.add_new_words(frame, t)
        assert eng.nn_last_kernel == 1
        assert np.array_equal(g, w), f"frame {t}"
        if t == 3:  # forget some indexed words: the compaction rebuilds the image
            victims = np.asarray(ids[100:140])
            eng.remove_words(victims)
            o.remove_words(victims)
    q = noisy(vocab[rng.integers(0, 6000, 50)], 0.05, rng)
    q[:10] = frame[150:160]                                  # descriptors that became words in the last frame (still not indexed)
    assert np.array_equal(eng.find_nn(q, True, 0.8), o.find_nn(q))
    # findNN searched the not-indexed words too (their rows are in the cached image now); the index-only search must not see them
    for a, b in zip(eng.knn2(q), o.knn2(q)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    eng.update()
    o.update()
    assert np.array_equal(eng.find_nn(q, True, 0.8), o.find_nn(q))
