"""Word-range sharding of FLOAT-descriptor dictionaries, host side (CPU only).

Each shard answers the 2-NN of every query over its own rows with the oracle's rtflann-order squared-L2 scan; the answers are packed as
64-bit keys (float bits of the distance << 32 | GLOBAL row, sharding.pack_keys_f32) and merged with sharding.merge_top2.  The merged
pair must equal the unsharded top-2 exactly: same distances, and on equal distances the lowest global row, as rtflann resolves ties."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import sharding, synth


def _sharded_top2(vocab, q, bounds):
    """bounds: [(r0, r1)] row ranges of the shards, in rank order -> merged [nq, 2] uint64 keys"""
    keys = []
    for r0, r1 in bounds:
        if r1 > r0:
            idx, dd = orc.knn2_raw(vocab[r0:r1], q)
            keys.append(sharding.pack_keys_f32(dd, np.where(idx >= 0, idx + r0, -1)))
        else:   # a rank without rows contributes no neighbour
            keys.append(np.full((len(q), 2), sharding.KEY64_NONE, np.uint64))
    return sharding.merge_top2(np.stack(keys))


def _unsharded_top2(vocab, q):
    idx, dd = orc.knn2_raw(vocab, q)
    return sharding.pack_keys_f32(dd, idx)


def _queries(vocab, n, seed):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, len(vocab), n)
    q = vocab[src] + rng.normal(0, 0.02, (n, vocab.shape[1])).astype(np.float32)
    q[: n // 4] = vocab[src[: n // 4]]                                           # distance 0
    q[n - n // 5:] = synth.make_float_vocabulary(n // 5, vocab.shape[1], seed + 1)  # unrelated descriptors
    return np.ascontiguousarray(q, np.float32)


def test_pack_keys_f32_orders_by_distance_then_row():
    d = np.array([[0.0, 0.0], [0.5, 0.25], [1e-30, 3.0e38]], np.float32)
    r = np.array([[7, 3], [0, 1 << 22], [5, -1]])
    k = sharding.pack_keys_f32(d, r)
    assert k.dtype == np.uint64
    assert k[0, 1] < k[0, 0] and k[1, 1] < k[1, 0] and k[2, 1] == sharding.KEY64_NONE
    assert int(k[1, 1]) & 0xFFFFFFFF == 1 << 22
    assert np.array_equal((k[:2] >> np.uint64(32)).astype(np.uint32).view(np.float32), d[:2])


@pytest.mark.parametrize("dim", [64, 128])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_merged_shard_keys_equal_the_unsharded_top2(dim, world):
    W = 1500
    vocab = synth.make_float_vocabulary(W, dim, 21)
    # exact duplicate rows on both sides of every shard edge: the lower global row must win
    edges = [sharding.shard_rows(W, world, r)[0] for r in range(1, world)]
    for e in edges:
        vocab[e] = vocab[e - 1]
    q = _queries(vocab, 120, 5)
    q[:len(edges)] = vocab[edges]          # queries that hit the duplicated pairs at distance 0
    bounds = [sharding.shard_rows(W, world, r) for r in range(world)]
    got = _sharded_top2(vocab, q, bounds)
    want = _unsharded_top2(vocab, q)
    assert np.array_equal(got, want)
    for i, e in enumerate(edges):
        assert int(got[i, 0]) == e - 1 and int(got[i, 1]) == e          # (0.0, row e-1), (0.0, row e)
    assert (got[:, 0] >> np.uint64(32) == 0).sum() >= 120 // 4          # the distance-0 queries stayed at distance 0


def test_one_row_shard_and_duplicates_across_it():
    W, dim = 400, 64
    vocab = synth.make_float_vocabulary(W, dim, 3)
    vocab[201] = vocab[200]      # the one-row shard [200, 201) holds a copy of the first row of the next shard
    vocab[199] = vocab[200]      # and of the last row of the previous one
    bounds = [(0, 200), (200, 201), (201, W)]
    q = _queries(vocab, 64, 8)
    q[0] = vocab[200]
    q[1] = vocab[200] + np.float32(1e-3)
    got = _sharded_top2(vocab, q, bounds)
    assert np.array_equal(got, _unsharded_top2(vocab, q))
    assert int(got[0, 0]) == 199 and int(got[0, 1]) == 200       # rows 199, 200, 201 tie at 0: the two lowest win
    # a one-row dictionary alone: its second neighbour is absent
    alone = _sharded_top2(vocab[200:201], q, [(0, 1)])
    assert (alone[:, 1] == sharding.KEY64_NONE).all() and np.array_equal(alone, _unsharded_top2(vocab[200:201], q))


def test_more_ranks_than_rows():
    """8 ranks over 5 rows: three ranks own nothing, the others one row each."""
    W, dim, world = 5, 128, 8
    vocab = synth.make_float_vocabulary(W, dim, 4)
    vocab[3] = vocab[2]
    bounds = [sharding.shard_rows(W, world, r) for r in range(world)]
    assert sum(1 for a, b in bounds if b == a) == 3
    q = _queries(vocab, 20, 9)
    q[0] = vocab[2]
    got = _sharded_top2(vocab, q, bounds)
    assert np.array_equal(got, _unsharded_top2(vocab, q))
    assert int(got[0, 0]) == 2 and int(got[0, 1]) == 3
    # fewer rows than two in the whole dictionary: the pair keeps its empty slot
    one = _sharded_top2(vocab[:1], q, [sharding.shard_rows(1, 3, r) for r in range(3)])
    assert (one[:, 1] == sharding.KEY64_NONE).all() and np.array_equal(one, _unsharded_top2(vocab[:1], q))
