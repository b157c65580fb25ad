"""256-D float descriptors (SuperPoint) without a GPU: the oracle's 2-NN against the reference's own rtflann, the database round trip of
1 KB float Word blobs, and lcd_create's width check, which runs before it looks for a device."""
from pathlib import Path

import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, LcdError, dbio
from rtabmap_b200.capi import LCD_DESC_F32

GOLDEN = Path(__file__).parent / "golden" / "ref_knn2_f256.npz"


def knn2_case(rows, seed):
    """Unit rows with exact duplicates (ties -> lowest row), queries near rows, on rows and far from every row."""
    rng = np.random.default_rng(seed)
    data = rng.standard_normal((rows, 256)).astype(np.float32)
    data /= np.linalg.norm(data, axis=1, keepdims=True)
    q = (data[rng.integers(0, rows, 48)] + 0.02 * rng.standard_normal((48, 256))).astype(np.float32)
    if rows > 10:
        data[7] = data[2]
        data[rows - 1] = data[2]
        q[0] = data[2]
        q[1] = data[rows - 2]
    q[2] = 3.0
    return data, q


CASES = [(1, 1), (2, 2), (700, 3), (1500, 4)]


@pytest.mark.parametrize("rows,seed", CASES)
def test_l2_256_matches_rtflann_bit_exact(rows, seed):
    """The oracle's 2-NN (the GPU tests' reference at 256-D) returns the ids and distance bits of rtflann's LinearIndex.  The rtflann
    answers are stored in tests/golden/ref_knn2_f256.npz and also recomputed where oracle/_ref/libref_flann.so has been built."""
    data, q = knn2_case(rows, seed)
    stored = np.load(GOLDEN)
    i_ref, d_ref = stored[f"idx_{rows}"].astype(np.int64), stored[f"dist_{rows}"]
    if orc.ref_lib() is not None:
        i_live, d_live = orc.ref_knn2(data, q)
        assert np.array_equal(i_live, i_ref) and np.array_equal(d_live.view(np.uint32), d_ref.view(np.uint32)), "stored answer is stale"
    i_orc, d_orc = orc.knn2_raw(data, q)
    assert np.array_equal(i_ref, i_orc)
    valid = i_ref >= 0
    assert np.array_equal(d_ref[valid].view(np.uint32), d_orc[valid].view(np.uint32))
    if rows > 10:
        assert tuple(i_orc[0]) == (2, 7)


def test_dbio_round_trip_of_256_float_words(tmp_path):
    """Word blobs of 1024 bytes with descriptor_size 256 are float rows (VWDictionary's CV_32F case), read and written back unchanged."""
    import sqlite3

    from test_dbio import make_db

    rng = np.random.default_rng(5)
    ids = np.sort(rng.choice(np.arange(1, 900), 200, replace=False)).astype(np.int32)
    desc = rng.standard_normal((200, 256)).astype(np.float32)
    db = str(tmp_path / "superpoint.db")
    make_db(db, ids, desc, [])
    con = sqlite3.connect(db)
    assert {(int(s), len(b)) for s, b in con.execute("SELECT descriptor_size, descriptor FROM Word")} == {(256, 1024)}
    con.close()
    got = dbio.read_dictionary(db)
    assert got.descriptors.dtype == np.float32 and got.descriptors.shape == (200, 256)
    assert np.array_equal(got.ids, ids) and np.array_equal(got.descriptors.view(np.uint32), desc.view(np.uint32))
    more_ids = np.array([1000, 1001], np.int32)
    more = rng.standard_normal((2, 256)).astype(np.float32)
    dbio.write_dictionary(db, more_ids, more)
    again = dbio.read_dictionary(db)
    assert np.array_equal(again.ids, np.concatenate([ids, more_ids]))
    assert np.array_equal(again.descriptors[-2:].view(np.uint32), more.view(np.uint32)) and again.last_word_id == 1001


@pytest.mark.parametrize("dim", [0, 32, 200, 255, 257, 512])
def test_float_widths_other_than_64_128_256_are_refused(dim):
    with pytest.raises(LcdError, match="float descriptors must have 64, 128 or 256 dimensions"):
        Engine(desc_type=LCD_DESC_F32, desc_dim=dim)


def test_256_float_width_passes_the_width_check():
    """lcd_create checks the width before it looks for a device: without one, a 256-D config fails only for the missing device."""
    try:
        eng = Engine(desc_type=LCD_DESC_F32, desc_dim=256)
    except LcdError as err:
        assert "no usable CUDA device" in str(err) and "dimensions" not in str(err)
    else:
        assert eng.desc_dim == 256
        eng.close()
