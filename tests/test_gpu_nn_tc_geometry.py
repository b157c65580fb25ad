"""The binary tensor-core 2-NN (nn_tensor.cuh) at the edges of its launch geometry: tiles of 256 queries (four consumer warpgroups of
64), word tiles searched as two half-tiles of 128 columns, and 16-bit epilogue keys that pair fragment columns i and i + 8 of one
half-tile (tile columns col and col + 64).

Every GPU case compares the tensor-core kernel and the POPC kernel with the exact fp64 reference of test_gpu_nn_edges key for key.  The
shapes come from a copy of run_knn's plan (engine.cu) for 256-query tiles, and each case asserts that it reaches the geometry it names.
The results do not depend on the geometry, so every case holds for any tile shape.

The CPU case replays the kernel's mbarrier arithmetic (stage, parity and arrival counts as functions of a CTA's running tile count)
over several items and a partly filled last word tile, with a producer and 16 consumer warps that run in every order.
"""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth
from test_gpu_nn_binary_mma import skewed_words
from test_gpu_nn_edges import (KEY_ROW_MASK, KEY_SHIFT, Mirror, binary_engine, check_both_kernels, flip_n, mixed_queries, ref_knn2_keys,
                               shard_keys, sm_count)

TC_BM, TC_BN, TC_HALF = 256, 256, 128   # nn_tensor.cuh: kTcBM, kTcBN, kTcHalfN
STAGES, CONSUMER_WARPS = 8, 16          # kTcStages; 4 consumer warpgroups of 4 warps


def tc_plan(n_rows: int, nq: int, sms: int, comm: bool = False) -> dict:
    """run_knn's split chooser and grid for the binary tensor-core kernel (engine.cu)."""
    n_wtiles, n_qtiles = -(-n_rows // TC_BN), -(-nq // TC_BM)
    best_split, best_cost = 1, -1
    for sp in range(1, min(n_wtiles, 16) + 1):
        tps = -(-n_wtiles // sp)
        if -(-n_wtiles // tps) != sp:
            continue
        cost = -(-(n_qtiles * sp) // sms) * (tps + 2)
        if best_cost < 0 or cost < best_cost:
            best_cost, best_split = cost, sp
    tps = -(-n_wtiles // best_split)
    n_items = n_qtiles * best_split
    grid = -(-n_items // max(1, min(8, -(-48 // max(tps, 1))))) if comm else min(n_items, sms)
    return dict(n_wtiles=n_wtiles, n_qtiles=n_qtiles, splits=best_split, tps=tps, n_items=n_items, grid=grid,
                max_items=-(-n_items // grid), min_items=n_items // grid, last_valid=n_rows - (n_wtiles - 1) * TC_BN)


def cta_tiles(plan: dict, cta: int, n_rows: int) -> list:
    """The word tiles CTA `cta` walks, item after item, as knn2_tensor_kernel's item_tiles gives them to every role."""
    tiles = []
    for item in range(cta, plan["n_items"], plan["grid"]):
        begin = (item // plan["n_qtiles"]) * plan["tps"]
        tiles += range(begin, min(plan["n_wtiles"], begin + plan["tps"]))
    return tiles


# ---------------------------------------------------------------- CPU: the barrier phases -------------------------------------------
class MBar:
    """mbarrier: a phase completes when `count` arrivals (and the expected bytes) have come; try_wait.parity(p) passes once the
    phase of parity p has completed, i.e. while the current phase's parity differs from p."""

    def __init__(self, count):
        self.count, self.pending, self.phase = count, 0, 0

    def arrive(self):
        self.pending += 1
        assert self.pending <= self.count
        if self.pending == self.count:
            self.pending, self.phase = 0, self.phase + 1

    def passes(self, parity):
        return (self.phase & 1) != parity


def run_phase_model(n_tiles: int, rng) -> None:
    """One producer thread and CONSUMER_WARPS consumer warps step through one CTA's tile stream in a random interleaving, with the
    kernel's waits and arrivals.  Every step must be able to proceed until all have finished (no hang), a consumer must read the tile
    the producer put in the stage for its running count g (no overtaking), and the producer must refill a stage only after every
    consumer warp released the tile before (no overwrite)."""
    full = [MBar(1) for _ in range(STAGES)]
    empty = [MBar(CONSUMER_WARPS) for _ in range(STAGES)]
    stage_tile = [None] * STAGES
    released = [0] * n_tiles
    prod, cons = 0, [0] * CONSUMER_WARPS

    def producer_step():
        nonlocal prod
        g, s = prod, prod % STAGES
        if g >= STAGES and not empty[s].passes(((g // STAGES) - 1) & 1):
            return False
        if g >= STAGES:
            assert released[g - STAGES] == CONSUMER_WARPS, f"stage {s} refilled before tile {g - STAGES} was released"
        stage_tile[s] = g
        full[s].arrive()   # arrive.expect_tx + the bulk copy's completion
        prod += 1
        return True

    def consumer_step(w):
        g = cons[w]
        s = g % STAGES
        if not full[s].passes((g // STAGES) & 1):
            return False
        assert stage_tile[s] == g, f"warp {w} read stage {s} holding tile {stage_tile[s]} for tile {g}"
        released[g] += 1
        empty[s].arrive()
        cons[w] += 1
        return True

    while prod < n_tiles or min(cons) < n_tiles:
        actors = [None] * (prod < n_tiles) + [w for w in range(CONSUMER_WARPS) if cons[w] < n_tiles]
        progressed = False
        for a in rng.permutation(len(actors)):
            a = actors[a]
            if producer_step() if a is None else consumer_step(a):
                progressed = True
                break
        assert progressed, f"hang: producer at tile {prod}, consumers at {cons}"
    assert released == [CONSUMER_WARPS] * n_tiles


@pytest.mark.parametrize("n_rows,nq,sms,comm", [
    (4097, 133 * TC_BM + 1, 132, False),    # 17 word tiles, several items per CTA, last word tile of one row
    (49152 + 129, 500 * TC_BM - 1, 132, False),
    (2049, 20000, 132, True),               # the word-range-sharded grid: many short items per CTA
    (2 * TC_BN + 127, 7 * TC_BM, 3, False),
])
def test_barrier_phases_over_several_items_and_a_partial_last_tile(n_rows, nq, sms, comm):
    rng = np.random.default_rng(n_rows + nq)
    plan = tc_plan(n_rows, nq, sms, comm)
    assert plan["min_items"] >= 2 and plan["last_valid"] < TC_BN, plan
    lengths = sorted({len(cta_tiles(plan, b, n_rows)) for b in range(plan["grid"])})
    assert lengths[-1] > STAGES, plan      # the ring wraps: every stage is reused with both parities
    for n in lengths[:1] + lengths[-1:]:
        for _ in range(3):
            run_phase_model(n, rng)


# ---------------------------------------------------------------- GPU cases --------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("short_by", [1, 0, -1], ids=["256k-1", "256k", "256k+1"])
def test_query_counts_around_a_multiple_of_the_query_tile(short_by):
    """nq = 256 k - 1, 256 k, 256 k + 1 with k = SMs + 1: the persistent grid walks several items per CTA, the last word split is
    short, and the last query tile is short by one, full, or holds one query."""
    sms = sm_count()
    n_rows = 4097
    nq = (sms + 1) * TC_BM - short_by
    plan = tc_plan(n_rows, nq, sms)
    assert plan["min_items"] >= 2 and plan["splits"] >= 2 and plan["tps"] * plan["splits"] > plan["n_wtiles"], plan
    assert nq - (plan["n_qtiles"] - 1) * TC_BM == {1: TC_BM - 1, 0: TC_BM, -1: 1}[short_by], plan
    rng = np.random.default_rng(nq)
    vocab = synth.make_binary_vocabulary(n_rows, 32, 11)
    ids = np.arange(1, n_rows + 1, dtype=np.int32) * 7
    check_both_kernels(binary_engine(vocab, ids), vocab, ids, mixed_queries(vocab, nq, rng), f"{nq} queries, {plan}")


@pytest.mark.gpu
@pytest.mark.parametrize("last_valid", [1, 127, 128, 129, 255, 256])
def test_last_word_tile_with_empty_partial_and_full_half_tiles(last_valid):
    """n_rows = 512 + last_valid: the last word tile's second half-tile is empty (1, 127, 128), partly valid (129, 255) or the tile is
    full (256).  Neighbours are planted on the last rows of the first half, the first rows of the second and the very last row."""
    n_rows = 2 * TC_BN + last_valid
    plan = tc_plan(n_rows, 5 * TC_BM + 3, sm_count())
    assert plan["last_valid"] == last_valid, plan
    rng = np.random.default_rng(last_valid)
    vocab = rng.integers(0, 256, (n_rows, 32), dtype=np.uint8)
    last0 = 2 * TC_BN
    plants = sorted({r for r in (last0, last0 + TC_HALF - 1, last0 + TC_HALF, last0 + TC_HALF + 1, n_rows - 1, n_rows - 2) if last0 <= r < n_rows})
    q = mixed_queries(vocab, 5 * TC_BM + 3, rng)
    for i, r in enumerate(plants):
        t = rng.integers(0, 256, 32, dtype=np.uint8)
        vocab[r] = flip_n(t, 1 + i % 3, rng)
        q[i * 37] = t
        q[i * 37 + 1] = vocab[r]
    ids = np.arange(1, n_rows + 1, dtype=np.int32)
    check_both_kernels(binary_engine(vocab, ids), vocab, ids, q, f"{n_rows} rows, {plan}")


@pytest.mark.gpu
def test_ties_across_half_tiles_and_packed_column_pairs():
    """Equal distances on tile columns c and c + 128 (the two half-tiles), on c and c + 64 (one 16-bit register pair of the epilogue),
    on 127 / 128 (last column of one half, first of the next) and 255 / 256 (across word tiles): the lower row wins every time."""
    n_rows = 6 * TC_BN + 77
    rng = np.random.default_rng(128)
    vocab = rng.integers(0, 256, (n_rows, 32), dtype=np.uint8)
    pairs = [(TC_BN + c, TC_BN + c + 128) for c in (0, 5, 66, 127)]
    pairs += [(2 * TC_BN + c, 2 * TC_BN + c + 64) for c in (0, 3, 63, 130, 191)]
    pairs += [(3 * TC_BN + 127, 3 * TC_BN + 128), (4 * TC_BN - 1, 4 * TC_BN), (5 * TC_BN + 128, 5 * TC_BN + 127), (6 * TC_BN + 10, 6 * TC_BN + 74)]
    groups = []
    for i, (a, b) in enumerate(pairs):
        t = rng.integers(0, 256, 32, dtype=np.uint8)
        d = i % 4
        vocab[a] = flip_n(t, d, rng) if d else t
        vocab[b] = flip_n(t, d, rng) if d else t
        groups.append((t, sorted((a, b)), d))
    q = mixed_queries(vocab, 3 * TC_BM, rng)
    pos = rng.permutation(len(q))[: 4 * len(groups)].reshape(len(groups), 4)   # every group at 4 query rows (warpgroups, lanes)
    for (t, _, _), rows in zip(groups, pos):
        q[rows] = t
    ref = ref_knn2_keys(vocab, q)
    for (t, rows_ab, d), rows in zip(groups, pos):
        got = [(int(k & KEY_ROW_MASK), int(k >> KEY_SHIFT)) for k in ref[rows[0]]]
        assert got == [(rows_ab[0], d), (rows_ab[1], d)], f"plant {rows_ab}: reference gives {got}"
    ids = np.arange(1, n_rows + 1, dtype=np.int32) * 3
    check_both_kernels(binary_engine(vocab, ids), vocab, ids, q, "planted ties across half-tiles")


@pytest.mark.gpu
@pytest.mark.parametrize("n_rows", [3 * TC_BN, 3 * TC_BN - 100], ids=["full_tiles", "last_tile_partial"])
def test_empty_and_full_queries_against_words_of_extreme_popcounts_in_both_halves(n_rows):
    """pa = 0 and pa = 256 make the distance pw and 256 - pw: the pw fields of T decide alone.  Words of popcount 1..12 and 244..255
    sit in both half-tiles of every tile (and in both half-words of a register pair), with repeated popcounts so ties decide too;
    random queries of low and high popcount see the same words, for which the AND count misleads."""
    rng = np.random.default_rng(n_rows)
    vocab = rng.integers(0, 256, (n_rows, 32), dtype=np.uint8)
    for r in rng.choice(n_rows, 120, replace=False):
        k = int(rng.integers(1, 13))
        bits = np.zeros(256, np.uint8)
        bits[rng.choice(256, k, replace=False)] = 1
        vocab[r] = np.packbits(bits) if rng.random() < 0.5 else ~np.packbits(bits)
    zeros, ones = np.zeros(32, np.uint8), np.full(32, 255, np.uint8)
    low = np.packbits(rng.random((100, 256)) < 0.05, axis=1)
    q = np.concatenate([np.stack([zeros, ones] * 64), low, ~low, skewed_words(100, rng)])
    ids = np.arange(1, n_rows + 1, dtype=np.int32)
    want = check_both_kernels(binary_engine(vocab, ids), vocab, ids, q, f"{n_rows} rows of extreme popcounts")
    pw = np.unpackbits(vocab, axis=1).sum(axis=1)
    for qi, dist in ((0, pw), (1, 256 - pw)):
        order = np.lexsort((np.arange(n_rows), dist))[:2]
        assert (want[0][qi], want[2][qi]) == (ids[order[0]], ids[order[1]])


@pytest.mark.gpu
def test_shard_keys_under_a_row_offset_on_the_sharded_grid():
    """lcd_shard_knn2_keys_dev with row_offset = 1 000 003 on an engine with a one-rank communicator, where the grid gives each CTA
    several short items; and the same keys without the communicator."""
    n_rows, nq, off = 513, 3000, 1_000_003
    plan = tc_plan(n_rows, nq, sm_count(), comm=True)
    assert plan["min_items"] >= 2 and plan["last_valid"] == 1, plan
    rng = np.random.default_rng(513)
    vocab = synth.make_binary_vocabulary(n_rows, 32, 5)
    vocab[TC_BN + 128] = vocab[TC_BN]             # a tie across the half-tiles of tile 1
    q = mixed_queries(vocab, nq, rng)
    q[::101] = vocab[TC_BN]
    want = ref_knn2_keys(vocab, q, row_offset=off)
    assert ((want[::101, 1] & KEY_ROW_MASK) == off + TC_BN + 128).all()
    ids = np.arange(1, n_rows + 1, dtype=np.int32)
    for comm in (False, True):
        eng = binary_engine(vocab, ids)
        if comm:
            eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        try:
            for kernel in (1, 0):
                eng.nn_select(kernel)
                eng.shard_set_row_offset(off)
                got = shard_keys(eng, q)
                assert eng.nn_last_kernel == kernel
                bad = np.flatnonzero((got != want).any(axis=1))
                assert bad.size == 0, f"communicator {comm}, kernel {kernel}: {bad.size} queries differ, first {bad[:4].tolist()}"
        finally:
            if comm:
                eng.shard_comm_destroy()


@pytest.mark.gpu
def test_cached_image_rebuilt_in_the_half_tile_layout_after_growth_removal_and_reordering():
    """The cached word image (rows and T) is rewritten only from the first tile that gained rows: after growth within and across
    half-tiles, removals that shift rows from one half-tile into the other, and out-of-order ids, every search sees the current rows."""
    rng = np.random.default_rng(640)
    pool = synth.make_binary_vocabulary(2000, 32, 640)
    pool[1::2] = ~pool[::2]                       # neighbouring rows of opposite popcount: a stale T after a shift is far off
    m = Mirror(Engine(), orc.OracleDictionary(0, 32, True, 0.8, True))
    used = 0

    def take(n):
        nonlocal used
        used += n
        return pool[used - n:used]

    def queries(n=900):
        return mixed_queries(np.stack([d for i, d in m.desc.items() if m.eng.has_word(i)]), n, rng)

    m.add(np.arange(1, 101) * 2, take(100))         # the first half-tile only
    m.update()
    m.check(queries(), "100 words: second half-tile empty")
    m.add(np.arange(101, 201) * 2, take(100))       # pending rows fill into the second half-tile
    q = queries()
    m.check_find_nn(q, "pending words in the second half-tile")
    m.check(q, "after findNN cached them")
    m.update()
    m.add(np.arange(201, 701) * 2, take(500))
    m.update()
    m.check(queries(), "grown to 700 rows")
    m.remove(np.concatenate([np.arange(1, 30) * 2, rng.choice(np.arange(30, 701) * 2, 70, replace=False)]).astype(np.int32))
    m.update()
    m.check(queries(), "removals: rows moved across half-tiles")
    m.add(np.arange(900, 1000)[::-1].copy() * 2, take(100))
    m.add(np.arange(701, 760) * 2, take(59))
    q = queries()
    m.check_find_nn(q, "out-of-order pending words")
    m.update()
    m.check(q, "out-of-order words indexed")
