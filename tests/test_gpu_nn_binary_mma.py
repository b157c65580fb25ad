"""The binary tensor-core 2-NN (nn_tensor.cuh) computes c = popc(q AND w) and orders the words of a query row by pw - 2 c, with the
per-word popcount pw cached beside the packed words of every 256-row tile.  These cases target what that encoding adds: words whose
popcounts differ sharply inside one tile (so that c alone would pick the wrong words), queries with no and with every bit set, and
the cached popcounts after the dictionary changes under them.  Every case compares the tensor-core kernel and the POPC kernel with the
exact reference, neighbour by neighbour.
"""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine
from test_gpu_nn_edges import TC_BN, Mirror, binary_engine, check_both_kernels, ref_knn2_keys

pytestmark = pytest.mark.gpu


def popcount(desc: np.ndarray) -> np.ndarray:
    return np.unpackbits(np.ascontiguousarray(desc, np.uint8), axis=1).sum(axis=1)


def skewed_words(n: int, rng) -> np.ndarray:
    """Rows whose popcounts spread over the whole [0, 256]: each row sets its bits with its own probability."""
    p = rng.uniform(0.0, 1.0, n)
    return np.packbits(rng.random((n, 256)) < p[:, None], axis=1)


def subset(desc: np.ndarray, drop: int, rng) -> np.ndarray:
    """desc with `drop` of its set bits cleared."""
    bits = np.unpackbits(desc[None].copy(), axis=1)[0]
    bits[rng.choice(np.flatnonzero(bits), drop, replace=False)] = 0
    return np.packbits(bits)


def superset(desc: np.ndarray, add: int, rng) -> np.ndarray:
    """desc with `add` of its clear bits set."""
    bits = np.unpackbits(desc[None].copy(), axis=1)[0]
    bits[rng.choice(np.flatnonzero(bits == 0), add, replace=False)] = 1
    return np.packbits(bits)


@pytest.mark.parametrize("n_rows", [4 * TC_BN, 4 * TC_BN - 37], ids=["full_tiles", "last_tile_partial"])
def test_popcounts_that_mislead_the_and_count_within_one_tile(n_rows):
    """Per planted query t (popcount ~128): a subset of t at distance 6-9 is its nearest word, while supersets of t in the same tile
    share more set bits with it (c = popc(t), larger than the subset's) at distances 10-40.  A kernel that ordered by c alone, or
    applied the wrong word's pw, would return a superset."""
    rng = np.random.default_rng(n_rows)
    vocab = skewed_words(n_rows, rng)
    queries, cases = [], []
    for tile in range(-(-n_rows // TC_BN)):
        lo, hi = tile * TC_BN, min(n_rows, (tile + 1) * TC_BN)
        picks = rng.choice(np.arange(lo, hi), 36, replace=False).reshape(6, 6)   # different lane quads and halves of the tile
        for rows in picks:
            t = np.packbits(rng.random(256) < 0.5)
            vocab[rows[0]] = subset(t, int(rng.integers(6, 10)), rng)
            vocab[rows[1]] = subset(t, 9, rng)
            for r in rows[2:]:
                vocab[r] = superset(t, int(rng.integers(10, 41)), rng)
            queries.append(t)
            cases.append(rows)
    q = np.stack(queries)
    ref = ref_knn2_keys(vocab, q)
    c = np.unpackbits(q[:, None, :] & vocab[None, :, :], axis=2).sum(axis=2)
    for i, rows in enumerate(cases):
        nearest = int(ref[i, 0] & ((1 << 22) - 1))
        assert nearest in rows[:2], f"query {i}: the planted subset is not the nearest word"
        assert c[i, rows[2:]].min() > c[i, nearest], f"query {i}: the supersets do not share more bits than the nearest word"
    q = np.concatenate([q, skewed_words(300, rng)])                # and queries of every popcount against the same words
    ids = np.arange(1, n_rows + 1, dtype=np.int32) * 5
    check_both_kernels(binary_engine(vocab, ids), vocab, ids, q, f"{n_rows} rows of skewed popcounts")


@pytest.mark.parametrize("n_rows", [TC_BN, TC_BN + 200], ids=["one_full_tile", "full_and_partial_tile"])
def test_queries_with_no_and_every_bit_set(n_rows):
    """pa = 0 and pa = 256 against words of every popcount 0..256: the distance is pw and 256 - pw, ties to the lowest row."""
    rng = np.random.default_rng(n_rows + 1)
    vocab = skewed_words(n_rows, rng)
    for k in range(min(n_rows, 257)):
        bits = np.zeros(256, np.uint8)
        bits[rng.choice(256, k, replace=False)] = 1
        vocab[(k * 97) % n_rows] = np.packbits(bits)                # popcount k, spread over lane quads and halves
    zeros, ones = np.zeros(32, np.uint8), np.full(32, 255, np.uint8)
    q = np.concatenate([np.stack([zeros, ones] * 70), skewed_words(57, rng)])
    ids = np.arange(1, n_rows + 1, dtype=np.int32)
    want = check_both_kernels(binary_engine(vocab, ids), vocab, ids, q, f"{n_rows} rows, empty and full queries")
    pw = popcount(vocab)
    for qi, dist in ((0, pw), (1, 256 - pw)):
        order = np.lexsort((np.arange(n_rows), dist))[:2]
        assert (want[0][qi], want[1][qi], want[2][qi], want[3][qi]) == (ids[order[0]], dist[order[0]], ids[order[1]], dist[order[1]])


def test_cached_popcounts_follow_removal_reordering_and_growth():
    """The popcounts live in the cached word image and are rewritten with the rows: after growth across a tile boundary (pending and
    indexed), after removals that shift rows onto other columns, and after out-of-order ids re-sort the pending rows."""
    rng = np.random.default_rng(256)
    pool = skewed_words(3000, rng)
    pool[1::2] = ~pool[::2]          # neighbouring rows of opposite popcount: a stale pw after a shift is far off
    m = Mirror(Engine(), orc.OracleDictionary(0, 32, True, 0.8, True))
    used = 0

    def take(n):
        nonlocal used
        used += n
        return pool[used - n:used]

    def queries(n=700):
        near = np.stack([d for i, d in m.desc.items() if m.eng.has_word(i)])
        q = near[rng.integers(0, len(near), n)]
        flip = rng.random(q.shape) < 0.02
        q = np.where(flip, q ^ np.uint8(1 << int(rng.integers(0, 8))), q)
        q[:3] = [np.zeros(32, np.uint8), np.full(32, 255, np.uint8), near[0]]
        return q

    m.add(np.arange(1, 251) * 2, take(250))
    m.update()
    m.check(queries(), "250 words: one partial tile")
    m.add(np.arange(251, 301) * 2, take(50))            # pending rows cross into the second tile
    q = queries()
    m.check_find_nn(q, "50 pending words across the tile boundary")
    m.check(q, "after findNN cached the pending rows")
    m.update()
    m.check(queries(), "pending words indexed across the tile boundary")
    m.add(np.arange(301, 1101) * 2, take(800))
    m.update()
    m.check(queries(), "grown to 1100 rows")
    m.remove(np.concatenate([np.arange(1, 40) * 2, rng.choice(np.arange(40, 1101) * 2, 60, replace=False)]).astype(np.int32))
    m.update()
    m.check(queries(), "low rows removed: every later row moved to another column")
    m.add(np.arange(1200, 1300)[::-1].copy() * 2, take(100))   # ids arrive in descending order: sort_pending reorders them
    m.add(np.arange(1101, 1150) * 2, take(49))
    q = queries()
    m.check_find_nn(q, "out-of-order pending words")
    m.update()
    m.check(q, "out-of-order words indexed")
