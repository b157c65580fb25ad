"""The tensor-core dictionary 2-NN searches at production batch sizes and at their tile, split and key edges, neighbour by neighbour.

Binary descriptors (nn_tensor.cuh): every case compares the two neighbours and their distances of the wgmma kernel with an exact
reference that uses none of the project's kernels (``ref_knn2_keys``: +-1 dot products in fp64, packed keys, lowest row wins a tie)
and with the POPC kernel.  The shapes are chosen with a copy of run_knn's split chooser so that the persistent grid really walks
several (query tile, word split) items per CTA, and neighbours and ties are planted on the word tile edge, the split edge, the lo/hi
half of the fast epilogue, different lane quads and the last row of a partly filled tile, with queries on both sides of every
query-side boundary.

Float descriptors (nn_tensor_f32.cuh): the fp16 filter + exact re-rank must equal the exact CUDA-core kernel bit for bit (and the
rtflann-order oracle on a subset), at several query tiles and splits, and with thousands of queries redone by the exact fallback.
"""
import numpy as np
import pytest
import torch

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import LCD_DESC_F32, LcdError

pytestmark = pytest.mark.gpu

KEY_SHIFT = 22                      # common.cuh: key = (distance << 22) | global row
KEY_ROW_MASK = (1 << KEY_SHIFT) - 1
KEY_NONE = 0xFFFFFFFF               # no neighbour (fewer than two rows)
MAX_ROWS_PACKED = 1 << KEY_SHIFT
LCD_ERR_CAPACITY = -3               # include/lcd_b200.h
TC_BM, TC_BN = 128, 256             # nn_tensor.cuh: queries per tile, words per tile
TF_BM, TF_BN = 128, 256             # nn_tensor_f32.cuh
FB_QUERIES = 4                      # nn_tensor_f32.cuh: kFbQueries


# ---------------------------------------------------------------- exact reference ----------------------------------------------
def _pm1(desc: np.ndarray, device) -> torch.Tensor:
    """[n, B] uint8 descriptors -> [n, 8B] fp64 of +-1 (bit b -> 2b - 1)."""
    bits = np.unpackbits(np.ascontiguousarray(desc, np.uint8), axis=1)
    return torch.from_numpy(bits).to(device=device, dtype=torch.float64).mul_(2.0).sub_(1.0)


def ref_knn2_keys(words: np.ndarray, queries: np.ndarray, row_offset: int = 0, device="cuda", chunk: int = 2048) -> np.ndarray:
    """Exact Hamming 2-NN as packed keys: int64 [nq, 2] of (distance << 22) | (row_offset + row), KEY_NONE where there is no row.

    The dot product of two +-1 vectors of n bits is n - 2 * hamming, an integer that fp64 holds exactly whatever the summation order,
    so distance = (n - dot) / 2 is exact.  The smallest two keys are the two nearest rows with the lowest row first among equal
    distances: the order rtflann's result set produces when it scans rows in ascending order."""
    words = np.ascontiguousarray(words, np.uint8)
    queries = np.ascontiguousarray(queries, np.uint8)
    nq, n_rows, n_bits = len(queries), len(words), words.shape[1] * 8
    out = np.full((nq, 2), KEY_NONE, np.int64)
    if n_rows == 0 or nq == 0:
        return out
    w = _pm1(words, device)
    rows = torch.arange(row_offset, row_offset + n_rows, dtype=torch.float64, device=device)
    k = min(2, n_rows)
    for q0 in range(0, nq, chunk):
        q = _pm1(queries[q0:q0 + chunk], device)
        key = q @ w.T                                         # dot, exact
        key.neg_().add_(n_bits).mul_(0.5)                     # distance, exact
        key.mul_(float(1 << KEY_SHIFT)).add_(rows)            # (distance << 22) | row, exact below 2^53
        best = torch.topk(key, k, dim=1, largest=False, sorted=True).values
        out[q0:q0 + len(q), :k] = best.to(torch.int64).cpu().numpy()
    return out


def keys_to_knn2(keys: np.ndarray, row_ids: np.ndarray):
    """Packed keys [nq, 2] (rows from 0) -> what lcd_dict_knn2 returns: (id1, d1, id2, d2), id 0 / distance -1 for no neighbour."""
    none = keys == KEY_NONE
    rows = np.where(none, 0, keys & KEY_ROW_MASK)
    ids = np.where(none, 0, np.asarray(row_ids, np.int64)[rows] if len(row_ids) else 0).astype(np.int32)
    dist = np.where(none, -1.0, keys >> KEY_SHIFT).astype(np.float32)
    return ids[:, 0], dist[:, 0], ids[:, 1], dist[:, 1]


def assert_same_knn2(got, want, what):
    names = ("id1", "d1", "id2", "d2")
    for name, g, w in zip(names, got, want):
        bad = np.flatnonzero(np.asarray(g).view(np.uint32) != np.asarray(w).view(np.uint32))
        assert bad.size == 0, f"{what}: {name} differs for {bad.size} queries, first {bad[:8].tolist()}: got {np.asarray(g)[bad[:8]].tolist()} want {np.asarray(w)[bad[:8]].tolist()}"


# ---------------------------------------------------------------- launch geometry (copies of run_knn / tf_search) --------------
def sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def tc_plan(n_rows: int, nq: int, sms: int, comm: bool = False) -> dict:
    """run_knn's split chooser and grid for the binary tensor-core kernel (engine.cu)."""
    n_wtiles, n_qtiles = -(-n_rows // TC_BN), -(-nq // TC_BM)
    best_split, best_cost = 1, -1
    for sp in range(1, min(n_wtiles, 16) + 1):
        tps = -(-n_wtiles // sp)
        if -(-n_wtiles // tps) != sp:
            continue
        waves = -(-(n_qtiles * sp) // sms)
        cost = waves * (tps + 3)
        if best_cost < 0 or cost < best_cost:
            best_cost, best_split = cost, sp
    tps = -(-n_wtiles // best_split)
    n_items = n_qtiles * best_split
    if comm:
        per_cta = max(1, min(8, -(-96 // max(tps, 1))))
        grid = -(-n_items // per_cta)
    else:
        grid = min(n_items, sms)
    return dict(n_wtiles=n_wtiles, n_qtiles=n_qtiles, splits=best_split, tps=tps, n_items=n_items, grid=grid,
                max_items=-(-n_items // grid), min_items=n_items // grid)


def tf_plan(n_rows: int, nq: int, dim: int, sms: int) -> dict:
    """tf_search's query tiles and word splits for the float tensor-core filter (engine.cu)."""
    n_tiles, n_qtiles = -(-n_rows // TF_BN), -(-nq // TF_BM)
    tiles_l2 = max(1, (24 << 20) // (TF_BN * dim * 2))
    splits = max(-(-n_tiles // tiles_l2), -(-(2 * sms) // n_qtiles))
    splits = max(1, min(splits, n_tiles))
    tps = -(-n_tiles // splits)
    return dict(n_qtiles=n_qtiles, splits=-(-n_tiles // tps), tps=tps)


# ---------------------------------------------------------------- helpers ------------------------------------------------------
def binary_engine(vocab, ids):
    eng = Engine()
    eng.add_words(ids, vocab)
    eng.last_word_id = int(np.max(ids))
    eng.update()
    return eng


def check_both_kernels(eng, words, row_ids, q, what):
    """knn2 on the tensor-core kernel and on the POPC kernel == the exact reference, id for id and distance for distance."""
    want = keys_to_knn2(ref_knn2_keys(words, q), row_ids)
    eng.nn_select(1)
    t = eng.knn2(q)
    assert eng.nn_last_kernel == 1, f"{what}: the tensor-core kernel did not run"
    assert_same_knn2(t, want, f"{what} (tensor core)")
    eng.nn_select(0)
    p = eng.knn2(q)
    assert eng.nn_last_kernel == 0
    assert_same_knn2(p, want, f"{what} (POPC)")
    eng.nn_select(1)
    return want


def mixed_queries(vocab, nq, rng, p_flip=0.04):
    """Near copies of dictionary rows, exact copies and random descriptors (whose two neighbours often tie in distance)."""
    q = rng.integers(0, 256, (nq, vocab.shape[1]), dtype=np.uint8)
    k = nq * 3 // 5
    q[:k] = synth.flip_bits(vocab[rng.integers(0, len(vocab), k)], p_flip, rng)
    q[k:k + nq // 10] = vocab[rng.integers(0, len(vocab), nq // 10)]
    return q[rng.permutation(nq)]


def flip_n(desc: np.ndarray, n: int, rng) -> np.ndarray:
    """desc with exactly n of its bits flipped."""
    bits = np.unpackbits(desc[None].copy(), axis=1)
    bits[0, rng.choice(bits.shape[1], n, replace=False)] ^= 1
    return np.packbits(bits, axis=1)[0]


# ---------------------------------------------------------------- 1. multi-item persistent grid ---------------------------------
# (rows, query tiles as a function of the SM count, queries missing from the last query tile, least items per CTA the case must
# reach, what else the chooser must have picked)
MULTI_ITEM = [
    pytest.param(4097, lambda s: s + 1, 5, 2, "short_last_split", id="sm+1_qtiles-4097rows"),
    pytest.param(4097, lambda s: 2 * s + 1, 3, 2, "unequal_items", id="2sm+1_qtiles-4097rows"),
    pytest.param(49153, lambda s: 2 * s + 1, 100, 10, "short_last_split", id="2sm+1_qtiles-49153rows"),
    pytest.param(49152, lambda s: 1000, 0, 20, "bench", id="bench-128000x49152"),
]


@pytest.mark.parametrize("n_rows,qtiles,short_by,min_items,shape", MULTI_ITEM)
def test_persistent_grid_walks_several_items_per_cta(n_rows, qtiles, short_by, min_items, shape):
    """Unsharded, run_knn launches min(items, SMs) CTAs: each CTA re-expands its query tile at every item boundary, prefetches the
    next item's queries and carries barrier phases and its running tile count across items.  Every neighbour must still be exact."""
    sms = sm_count()
    nq = qtiles(sms) * TC_BM - short_by
    plan = tc_plan(n_rows, nq, sms)
    assert plan["min_items"] >= min_items, plan
    if shape == "short_last_split":
        assert plan["splits"] >= 2 and plan["tps"] * plan["splits"] > plan["n_wtiles"], plan
    elif shape == "unequal_items":
        assert plan["max_items"] > plan["min_items"], plan
    else:
        assert nq == 128000 and plan["splits"] >= 2, plan
    rng = np.random.default_rng(n_rows + nq)
    vocab = synth.make_binary_vocabulary(n_rows, 32, n_rows)
    ids = np.arange(1, n_rows + 1, dtype=np.int32) * 3
    eng = binary_engine(vocab, ids)
    q = mixed_queries(vocab, nq, rng)
    check_both_kernels(eng, vocab, ids, q, f"{n_rows} rows x {nq} queries, {plan}")


# ---------------------------------------------------------------- 2. planted neighbours and ties on every boundary ---------------
def plant_boundaries(n_rows: int, tps: int, n_splits: int, rng):
    """A random dictionary with groups of rows planted around one fresh descriptor each.  Returns (vocab, [(query, want)]):
    `want` = the (row, distance) pairs the group is built to produce, checked against the reference before the kernels run."""
    vocab = rng.integers(0, 256, (n_rows, 32), dtype=np.uint8)
    split_edge = tps * TC_BN                      # first row of split 1
    last_split = (n_splits - 1) * tps * TC_BN     # first row of the last (short) split
    groups = []

    def fresh():
        return rng.integers(0, 256, 32, dtype=np.uint8)

    def group(rows_dists):
        # one fresh descriptor t, rows at the given distances from it (distinct bit flips: equidistant rows are different words);
        # every random row is ~100 bits away, so the two planted rows nearest to t are its two neighbours
        t = fresh()
        for r, d in rows_dists:
            vocab[r] = flip_n(t, d, rng) if d else t
        groups.append((t, [(r, d) for d, r in sorted((d, r) for r, d in rows_dists)[:2]]))

    used = set()

    def pick(*rows):
        # the first of these rows that exists and no other group holds (the split geometry moves with the query count)
        for r in rows:
            if 0 <= r < n_rows and r not in used:
                used.add(r)
                return r
        raise AssertionError(f"no free row among {rows}")

    group([(pick(255), 0), (pick(256), 0)])                              # word tile edge
    group([(pick(split_edge - 1), 0), (pick(split_edge), 0)])            # last row of split 0, first row of split 1
    group([(pick(last_split - 1, split_edge - 2), 2), (pick(last_split, split_edge + 1), 1)])   # into the last, short split
    group([(pick(TC_BN + 127), 0), (pick(TC_BN + 128), 0)])              # tile columns 127 / 128: lo / hi half of the fast epilogue
    group([(pick(2 * TC_BN + 128), 0), (pick(2 * TC_BN + 127), 1)])
    group([(pick(3 * TC_BN + 1), 0), (pick(3 * TC_BN + 2), 0)])          # lane quads 0 / 1
    group([(pick(3 * TC_BN + 6), 3), (pick(3 * TC_BN + 15), 3), (pick(3 * TC_BN + 9), 3)])   # quads 3 / 3 / 0, d1 == d2 == 3
    group([(pick(n_rows - 1, n_rows - 2, n_rows - 5), 0), (pick(5), 0)])  # the last row of the partly filled tile
    group([(pick(last_split + 7, last_split + 1, n_rows - 3), 0), (pick(100), 1)])  # first neighbour in the last split
    # the second neighbour improves by exactly one bit in a later tile; equal distances later still lose to the lower row
    group([(pick(10), 0), (pick(20), 5), (pick(700), 4), (pick(1800), 4), (pick(n_rows - 2, n_rows - 4), 4)])
    group([(pick(40), 3), (pick(300), 3), (pick(1000), 2), (pick(split_edge + 3), 2)])
    group([(pick(90), 2), (pick(91), 2)])                                # two different words at the same distance
    return vocab, groups


@pytest.mark.parametrize("n_rows", [4097, 4351], ids=["last_tile_valid1", "last_tile_valid255"])
@pytest.mark.parametrize("multi_item", [False, True], ids=["one_item_per_cta", "several_items_per_cta"])
def test_planted_ties_and_distances_on_every_tile_boundary(n_rows, multi_item):
    sms = sm_count()
    rng = np.random.default_rng(n_rows * 7 + multi_item)
    n_groups = 12
    nq = (sms + 1) * TC_BM - 9 if multi_item else (n_groups + 1) * TC_BM - 9
    plan = tc_plan(n_rows, nq, sms)
    assert plan["splits"] >= 2 and plan["tps"] * plan["splits"] > plan["n_wtiles"], plan
    assert (plan["min_items"] >= 2) == multi_item, plan
    vocab, groups = plant_boundaries(n_rows, plan["tps"], plan["splits"], rng)
    assert len(groups) == n_groups
    # Latin square over the first n_groups query tiles: every group sits at every row of a query tile once (rows 63 / 64 between the
    # consumer warpgroups, r_lo / r_lo + 8 of every lane, 127 / 128 across the query-tile edge), next to different groups
    q = mixed_queries(vocab, nq, rng)
    pos = np.arange(n_groups * TC_BM)
    gid = (pos % TC_BM + pos // TC_BM) % n_groups
    q[pos] = np.stack([groups[g][0] for g in gid])
    q[-1] = groups[0][0]                             # and in the last, partly filled query tile
    ids = np.arange(1, n_rows + 1, dtype=np.int32)
    ref = ref_knn2_keys(vocab, q)
    for g, (_, want) in enumerate(groups):           # the plants produce the intended neighbours in the reference
        k = ref[np.flatnonzero(gid == g)[0]]
        got = [(int(x & KEY_ROW_MASK), int(x >> KEY_SHIFT)) for x in k]
        assert got == want, f"group {g}: reference {got}, planted {want}"
    eng = binary_engine(vocab, ids)
    check_both_kernels(eng, vocab, ids, q, f"planted groups, {plan}")


def test_extreme_distances_and_a_one_word_dictionary():
    """Distance 0 and 256 (all-zero / all-one descriptors and complements) through the fast epilogue and the partial tile, and a
    dictionary of one word (no second neighbour)."""
    rng = np.random.default_rng(3)
    zeros, ones = np.zeros(32, np.uint8), np.full(32, 255, np.uint8)
    t = rng.integers(0, 256, 32, dtype=np.uint8)
    for n_rows in (1, 2, 256, 257, 600):
        vocab = np.tile(ones, (n_rows, 1))
        if n_rows >= 257:
            vocab[255] = zeros
            vocab[n_rows - 1] = zeros
            vocab[128] = t
            vocab[200] = ~t
        q = np.stack([zeros, ones, t, ~t, np.tile(np.array([0x0F], np.uint8), 32)] * 60)
        q = np.concatenate([q, rng.integers(0, 256, (37, 32), dtype=np.uint8)])
        ids = np.arange(1, n_rows + 1, dtype=np.int32) * 2
        eng = binary_engine(vocab, ids)
        want = check_both_kernels(eng, vocab, ids, q, f"{n_rows} extreme rows")
        first = tuple(a[0] for a in want)                     # the all-zero query
        if n_rows == 1:
            assert first == (2, 256, 0, -1)
        elif n_rows <= 256:
            assert first == (2, 256, 4, 256)                  # every row at distance 256: the two lowest rows
        else:
            assert first == (256 * 2, 0, n_rows * 2, 0)       # rows 255 and n_rows - 1
            assert tuple(a[1] for a in want) == (2, 0, 4, 0)  # the all-one query: rows 0 and 1


# ---------------------------------------------------------------- 3. key packing under a row offset -----------------------------
def shard_keys(eng, q: np.ndarray) -> np.ndarray:
    nq = len(q)
    d_q = torch.from_numpy(np.ascontiguousarray(q).reshape(-1)).cuda()
    k = torch.zeros(nq * 2, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.shard_knn2_keys_dev(d_q.data_ptr(), nq, k.data_ptr())
    eng.synchronize()
    return k.cpu().numpy().view(np.uint32).astype(np.int64).reshape(nq, 2)


def _keys_on_both_kernels(eng, vocab, q, off, what):
    want = ref_knn2_keys(vocab, q, row_offset=off)
    assert int((want[:, 0] & KEY_ROW_MASK).max()) <= MAX_ROWS_PACKED - 1
    out = {}
    for kernel in (1, 0):
        eng.nn_select(kernel)
        eng.shard_set_row_offset(off)
        got = shard_keys(eng, q)
        assert eng.nn_last_kernel == kernel
        bad = np.flatnonzero((got != want).any(axis=1))
        assert bad.size == 0, f"{what}, kernel {kernel}: {bad.size} queries differ, first {bad[:4].tolist()}: {got[bad[:4]].tolist()} vs {want[bad[:4]].tolist()}"
        out[kernel] = got
        eng.shard_set_row_offset(MAX_ROWS_PACKED - len(vocab) + 1)
        with pytest.raises(LcdError) as err:
            shard_keys(eng, q)
        assert err.value.code == LCD_ERR_CAPACITY
    eng.nn_select(1)
    return out[1]


def test_keys_up_to_the_last_packed_row_under_a_row_offset():
    """row_offset + n_rows == 2^22: rows up to 2^22 - 1 come back with their distance field intact; one row more is refused.  Again
    on an engine with a one-rank communicator, where the search runs as a grid of several items per CTA."""
    n_rows, nq = 513, 3000
    rng = np.random.default_rng(22)
    vocab = synth.make_binary_vocabulary(n_rows, 32, 4)
    vocab[n_rows - 1] = vocab[3]                   # tie on the very last row: 2^22 - 1
    vocab[n_rows - 2] = ~vocab[3]
    ids = np.arange(1, n_rows + 1, dtype=np.int32)
    q = mixed_queries(vocab, nq, rng)
    q[::97] = vocab[3]
    q[1::97] = ~vocab[n_rows - 1]
    off = MAX_ROWS_PACKED - n_rows
    eng = binary_engine(vocab, ids)
    plain = _keys_on_both_kernels(eng, vocab, q, off, "no communicator")
    assert (plain[::97, 1] & KEY_ROW_MASK == MAX_ROWS_PACKED - 1).all()
    assert (plain[1::97, 0] >> KEY_SHIFT == 0).all()

    plan = tc_plan(n_rows, nq, sm_count(), comm=True)
    assert plan["min_items"] >= 2, plan
    eng2 = binary_engine(vocab, ids)
    eng2.shard_comm_init(Engine.shard_unique_id(), 0, 1)
    try:
        with_comm = _keys_on_both_kernels(eng2, vocab, q, off, "one-rank communicator")
    finally:
        eng2.shard_comm_destroy()
    assert np.array_equal(with_comm, plain)


# ---------------------------------------------------------------- 4. the cached word image across dictionary changes ------------
class Mirror:
    """The engine, the oracle and the descriptors of every word id, changed together."""

    def __init__(self, eng, o):
        self.eng, self.o, self.desc = eng, o, {}

    def add(self, ids, desc):
        ids = np.asarray(ids, np.int32)
        self.eng.add_words(ids, desc)
        self.o.add_words(ids, desc)
        self.desc.update({int(i): d for i, d in zip(ids, desc)})
        last = max(self.o.last_word_id, int(ids.max()))
        self.eng.last_word_id = last
        self.o.last_word_id = last

    def remove(self, ids):
        self.eng.remove_words(ids)
        self.o.remove_words(ids)

    def update(self):
        self.eng.update()
        self.o.update()

    def indexed(self):
        ids = self.o.indexed_ids()
        assert np.array_equal(self.eng.get_indexed()[0], ids)
        return ids, np.stack([self.desc[int(i)] for i in ids])

    def check(self, q, what):
        ids, words = self.indexed()
        check_both_kernels(self.eng, words, ids, q, what)

    def check_find_nn(self, q, what):
        want = self.o.find_nn(q)
        for kernel in (1, 0):
            self.eng.nn_select(kernel)
            assert np.array_equal(self.eng.find_nn(q, True, 0.8), want), f"{what}: find_nn, kernel {kernel}"
        self.eng.nn_select(1)


def test_cached_word_image_follows_every_dictionary_change():
    """The +-1 image of the words is cached with the dictionary and only rewritten from the first changed tile: after each change
    the search must see exactly the current rows."""
    rng = np.random.default_rng(71)
    pool = synth.make_binary_vocabulary(12000, 32, 71)
    m = Mirror(Engine(), orc.OracleDictionary(0, 32, True, 0.8, True))
    used = 0

    def take(n):
        nonlocal used
        used += n
        return pool[used - n:used]

    def queries(n=1500):   # near the words in the dictionary now, indexed or pending
        return mixed_queries(np.stack([d for i, d in m.desc.items() if m.eng.has_word(i)]), n, rng)

    m.add(np.arange(1, 1001) * 2, take(1000))
    m.update()
    m.check(queries(), "1000 indexed words")
    # findNN with words pending: the pending rows join the cached image, the index-only search must not see them
    m.add(np.arange(1001, 1301) * 2, take(300))
    q = queries()
    m.check_find_nn(q, "300 pending words")
    m.check(q, "after findNN cached the pending rows")
    m.update()
    m.check(queries(), "pending words indexed")
    # grow the image past its reserve (16 tiles for the first 1000 rows): the cached tiles are carried over
    m.add(np.arange(1301, 5301) * 2, take(4000))
    m.update()
    m.check(queries(), "grown past the reserve")
    # remove indexed words: the rows are compacted at update()
    m.remove(rng.choice(np.arange(1, 5301) * 2, 50, replace=False).astype(np.int32))
    m.update()
    m.check(queries(), "indexed words removed")
    # remove a pending word after findNN cached it
    m.add(np.arange(5301, 5501) * 2, take(200))
    m.check_find_nn(queries(), "200 pending words")
    m.remove(np.array([5400 * 2], np.int32))
    q = queries()
    m.check_find_nn(q, "a pending word removed")
    m.update()
    m.check(q, "pending words indexed after a removal")
    # out-of-order ids: sort_pending moves rows that findNN already cached
    m.add(np.arange(6001, 6101) * 2, take(100))
    m.check_find_nn(queries(), "100 pending words")
    m.add((np.arange(5501, 5551) * 2)[::-1].copy(), take(50))
    q = queries()
    m.check_find_nn(q, "pending words re-sorted")
    m.update()
    m.check(q, "re-sorted pending words indexed")
    # clear() and a different vocabulary of the same size
    n = m.eng.indexed_size()
    m.eng.clear()
    m.o = orc.OracleDictionary(0, 32, True, 0.8, True)
    m.desc = {}
    other = synth.make_binary_vocabulary(n, 32, 72)
    m.add(np.arange(1, n + 1) * 2, other)
    m.update()
    m.check(queries(), "cleared and refilled with a different vocabulary")


# ---------------------------------------------------------------- 5. float descriptors: filter + re-rank, and the fallback -------
def float_vocab(n, dim, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, dim)).astype(np.float32)
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def noisy(rows, sigma, rng):
    q = rows + sigma * rng.standard_normal(rows.shape).astype(np.float32)
    return (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)


def float_engine(vocab):
    eng = Engine(desc_type=LCD_DESC_F32, desc_dim=vocab.shape[1])
    ids = np.arange(1, len(vocab) + 1, dtype=np.int32)
    eng.add_words(ids, vocab)
    eng.last_word_id = len(vocab)
    eng.update()
    return eng, ids


def tensor_vs_exact_float(eng, q):
    eng.nn_select(1)
    g = eng.knn2(q)
    assert eng.nn_last_kernel == 1, "the tensor-core filter did not run"
    stats = eng.nn_f32_stats(len(q))
    eng.nn_select(0)
    x = eng.knn2(q)
    assert eng.nn_last_kernel == 0
    eng.nn_select(1)
    assert_same_knn2(g, x, "float tensor filter vs the exact kernel")
    return g, stats


def test_float_filter_over_many_query_tiles_and_splits():
    dim, n_rows, nq = 64, 70001, 20000
    plan = tf_plan(n_rows, nq, dim, sm_count())
    assert plan["n_qtiles"] > 100 and plan["splits"] >= 2, plan
    vocab = float_vocab(n_rows, dim, 5)
    rng = np.random.default_rng(6)
    q = float_vocab(nq, dim, 7)
    q[: nq // 2] = noisy(vocab[rng.integers(0, n_rows, nq // 2)], 0.05, rng)
    q[nq // 2: nq // 2 + 500] = vocab[rng.integers(0, n_rows, 500)]
    q = q[rng.permutation(nq)]
    eng, ids = float_engine(vocab)
    g, _ = tensor_vs_exact_float(eng, q)
    o = orc.OracleDictionary(1, dim, True, 0.8, True)
    o.add_words(ids, vocab)
    o.update()
    sub = rng.choice(nq, 1000, replace=False)
    assert_same_knn2([a[sub] for a in g], o.knn2(q[sub]), "float tensor filter vs the oracle")


@pytest.mark.parametrize("n_fb,n_plain", [(1, 600), (2000, 500), (68000, 500)])
def test_float_fallback_redoes_thousands_of_overflowing_queries(n_fb, n_plain):
    """Queries whose nearest row sits in a block of 420 identical rows overflow their candidate list and are redone by the exact
    scan, which spreads them over S row-splits x query-group slots; with more than 2 * SMs * kFbQueries of them every slot loops
    over several groups, and past 65536 queries the scratch grows with the query count."""
    dim, n_rows = 64, 12000
    sms = sm_count()
    vocab = float_vocab(n_rows, dim, 31)
    block = slice(2000, 2420)
    vocab[block] = vocab[7]
    rng = np.random.default_rng(n_fb)
    # the other queries are near rows on the far side of the block (squared distance > 2.2 from it): the block can never be within
    # the filter's bound of their second neighbour (~1.2), so their lists stay short and exactly the intended queries fall back
    plain_rows = np.setdiff1d(np.flatnonzero(vocab @ vocab[7] < -0.1), np.r_[7, 2000:2420])
    q = np.concatenate([noisy(np.repeat(vocab[7:8], n_fb, 0), 0.02, rng), noisy(vocab[rng.choice(plain_rows, n_plain)], 0.03, rng)])
    perm = rng.permutation(len(q))
    q = q[perm]
    intended = perm < n_fb
    eng, ids = float_engine(vocab)
    g, (fb, n_cand, _) = tensor_vs_exact_float(eng, q)
    near_block = (g[0] == 8) & (g[2] == 2001)     # rows 7 and 2000: ties resolve to the lowest rows
    assert np.array_equal(near_block, intended)
    assert fb == n_fb, f"{fb} queries fell back, {n_fb} intended ({n_cand} candidates re-ranked)"
    if n_fb > 1:
        assert n_fb > 2 * sms * FB_QUERIES
    o = orc.OracleDictionary(1, dim, True, 0.8, True)
    o.add_words(ids, vocab)
    o.update()
    sub = np.concatenate([np.flatnonzero(intended)[:150], np.flatnonzero(~intended)[:50]])
    assert_same_knn2([a[sub] for a in g], o.knn2(q[sub]), "fallback vs the oracle")
