"""Host-side logic of word-range sharding across GPUs (SURVEY.md §8(e), BASELINE config 5).

Rank r of G owns a contiguous range of vocabulary rows (rows are in ascending word id, the
search order of VWDictionary::update) and the posting lists of exactly those words.  Every rank
brings its own frames.  Per step (lcd_shard_process_frames_dev / lcd_shard_localize_batch_dev):
  1. all-gather of the descriptors: every rank sees the frames of all ranks;
  2. every rank finds the local top-2 of each descriptor over its rows as packed keys with GLOBAL
     rows — binary: dist << 22 | row (u32), float: float bits of the squared distance << 32 | row
     (u64) — and an all-to-all sends each rank the keys of ITS frames;
  3. every rank merges the G key sets of its frames (unsigned min-2 = the reference's
     (distance, lowest row) order), runs the NNDR / new-word pass, and the word ids are all-gathered;
  4. every rank scores all frames over the words it owns into exact fixed-point int64 sums; a
     reduce-scatter leaves each rank the summed scores of its own frames.
No computation of the hot path happens here: this module only partitions inputs and packs keys
(the numpy merge below is the specification the CPU tests check the partitioning against).
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

KEY_SHIFT = 22
KEY_ROW_MASK = (1 << KEY_SHIFT) - 1
KEY_NONE = np.uint32(0xFFFFFFFF)
KEY64_NONE = np.uint64(0xFFFFFFFFFFFFFFFF)


def shard_rows(n_rows: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous, balanced row range [r0, r1) of `rank`."""
    base, rem = divmod(n_rows, world)
    r0 = rank * base + min(rank, rem)
    return r0, r0 + base + (1 if rank < rem else 0)


def shard_csr(word_ids: np.ndarray, row_ptr: np.ndarray, sig: np.ndarray, cnt: np.ndarray, owned_ids: np.ndarray):
    """Subset of a word-major CSR inverted index restricted to the words in `owned_ids`."""
    owned = np.isin(word_ids, owned_ids)
    lens = np.diff(row_ptr)
    keep = np.repeat(owned, lens)
    new_ptr = np.concatenate([[0], np.cumsum(lens[owned])]).astype(np.int64)
    return word_ids[owned], new_ptr, sig[keep], cnt[keep]


def pack_keys(dist: np.ndarray, row: np.ndarray) -> np.ndarray:
    return (dist.astype(np.uint32) << np.uint32(KEY_SHIFT)) | row.astype(np.uint32)


def pack_keys_f32(dist: np.ndarray, row: np.ndarray) -> np.ndarray:
    """Float-descriptor keys: (float32 bits of the squared distance << 32) | global row, uint64.  Distances are >= 0, so the unsigned
    order of the key is (distance, lowest row) order; a negative row (no neighbour) packs as KEY64_NONE."""
    dist = np.ascontiguousarray(dist, np.float32)
    row = np.asarray(row)
    rows = np.maximum(row, 0).astype(np.uint64)
    keys = (dist.view(np.uint32).astype(np.uint64) << np.uint64(32)) | rows
    return np.where(row >= 0, keys, KEY64_NONE).astype(np.uint64)


def merge_top2(keys: np.ndarray) -> np.ndarray:
    """keys [G, nq, 2] of an unsigned dtype -> [nq, 2]: the two smallest keys per query (all ones = absent)."""
    g, nq, _ = keys.shape
    flat = np.sort(np.transpose(keys, (1, 0, 2)).reshape(nq, g * 2), axis=1)
    return flat[:, :2]
