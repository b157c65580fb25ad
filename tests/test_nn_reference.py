"""The exact Hamming 2-NN reference of tests/test_gpu_nn_edges.py, pinned on the CPU to the oracle's restated rtflann linear scan:
a bug in the reference must not hide a bug in the kernels it checks."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import synth
from test_gpu_nn_edges import KEY_NONE, KEY_ROW_MASK, KEY_SHIFT, MAX_ROWS_PACKED, ref_knn2_keys


def oracle_keys(words, queries, row_offset=0):
    idx, dist = orc.knn2_raw(words, queries)
    keys = (dist.astype(np.int64) << KEY_SHIFT) | (idx.astype(np.int64) + row_offset)
    return np.where(idx < 0, KEY_NONE, keys)


@pytest.mark.parametrize("n_rows", [1, 2, 3, 257, 700])
def test_reference_equals_the_oracle_with_ties(n_rows):
    rng = np.random.default_rng(n_rows)
    words = synth.make_binary_vocabulary(n_rows, 32, n_rows + 1)
    if n_rows >= 257:
        words[255] = words[256] = words[17]          # three copies: the two lowest rows win
        words[100] = np.zeros(32, np.uint8)
        words[n_rows - 1] = np.full(32, 255, np.uint8)
        for r, bit in ((300 % n_rows, 1), (301 % n_rows, 2)):   # two different words one bit away from row 3
            words[r] = words[3]
            words[r, 0] ^= bit
    q = rng.integers(0, 256, (300, 32), dtype=np.uint8)
    q[:100] = synth.flip_bits(words[rng.integers(0, n_rows, 100)], 0.05, rng)
    q[100] = words[17 % n_rows]
    q[101] = words[3 % n_rows]
    q[102] = np.zeros(32, np.uint8)
    q[103] = np.full(32, 255, np.uint8)
    for off in (0, MAX_ROWS_PACKED - n_rows):
        got = ref_knn2_keys(words, q, row_offset=off, device="cpu", chunk=128)
        assert np.array_equal(got, oracle_keys(words, q, off))
    got = ref_knn2_keys(words, q, device="cpu")
    if n_rows == 1:
        assert (got[:, 1] == KEY_NONE).all() and (got[:, 0] & KEY_ROW_MASK == 0).all()
        assert got[102, 0] >> KEY_SHIFT == int(np.unpackbits(words[0]).sum())
    if n_rows >= 257:
        assert got[100].tolist() == [17, 255]
        assert got[101].tolist() == [3, (1 << KEY_SHIFT) | (300 % n_rows)]
        assert got[102, 0] == 100 and got[103, 0] == n_rows - 1
        assert (got[102, 1] >> KEY_SHIFT) > 0
