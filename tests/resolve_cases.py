"""Seeded frames and dictionaries that take the new-word loop of the quantiser (VWDictionary::addNewWords, resolve_rounds /
resolve_rounds_l2) to its edges: alternating chains that need every pass of a 32-descriptor chunk, ties in the multimap's insertion
order, NNDR products at the float boundary and frames up to the 4096-descriptor limit (test_oracle_resolve_cases.py,
test_gpu_resolve_edges.py)."""
from __future__ import annotations

import numpy as np

BIN_CHAINS = ((50, 16), (100, 32), (200, 64))     # (chain length, descriptor bytes)
F32_CHAINS = ((40, 64), (100, 128), (200, 256))   # (chain length, dimensions)
# rows of far descriptors before the chain: 0 puts it on chunk starts; 29 makes it straddle rows 32 and 64 with an odd chain
# position there, so lane 0 of those chunks matches the previous chunk's last word
LEADS = (0, 29)
TAIL = 7
MAX_FRAME = 4096
# (nndr, best, second, accepted by the reference's float product `best > nndr * second`)
NNDR_CASES = ((0.8, 8, 10, True), (0.8, 9, 11, False), (0.7, 7, 10, True))


def _pack(bits):
    return np.packbits(bits.astype(np.uint8), axis=-1)


def binary_chain(length: int, dim: int, seed: int):
    """(chain [length, dim], index words [2*length, dim]) uint8.  D_i is a random R with the 2-bit groups g_i and g_i+1 flipped, so
    d(D_i, D_i-1) = 4 and d(D_i, D_j) = 8 for |i - j| >= 2; each D_i has two index words 9 bits away in bits no group uses.  Quantised
    in order, the chain alternates: new word, match to the word just created, new word, ..."""
    rng = np.random.default_rng(seed)
    nbits = 8 * dim
    perm = rng.permutation(nbits)
    groups = perm[:2 * (length + 1)].reshape(length + 1, 2)
    free = perm[2 * (length + 1):]
    assert len(free) >= 9
    r = rng.integers(0, 2, nbits)
    chain = np.repeat(r[None], length, 0)
    for i in range(length):
        chain[i, groups[i]] ^= 1
        chain[i, groups[i + 1]] ^= 1
    index = np.repeat(chain, 2, 0)
    for k in range(2 * length):
        index[k, rng.choice(free, 9, replace=False)] ^= 1
    return _pack(chain), _pack(index)


def float_chain(length: int, dim: int, seed: int, a: float = 0.1):
    """(chain [length, dim], index words [2*length, dim]) float32: D_i = b + a (u_i + u_i+1) with the u orthonormal, so squared
    distances are 2a^2 to the neighbour and 4a^2 further along; the index words D_i +- sqrt(4.5) a v, v orthogonal to the chain's
    span, are 4.5a^2 away.  Alternates like binary_chain."""
    rng = np.random.default_rng(seed)
    assert length + 2 <= dim
    q, _ = np.linalg.qr(rng.standard_normal((dim, length + 2)))
    u, v = q[:, :length + 1].T, q[:, length + 1]
    b = rng.standard_normal(dim)
    b /= np.linalg.norm(b)
    chain = b + a * (u[:-1] + u[1:])
    off = np.sqrt(4.5) * a * v
    index = np.stack([chain + off, chain - off], 1).reshape(2 * length, dim)
    return chain.astype(np.float32), index.astype(np.float32)


def far_rows(n: int, dim: int, dtype, rng) -> np.ndarray:
    """Descriptors far from everything else: random bytes, or random unit vectors (a chain lies near one point)."""
    if dtype == np.uint8:
        return rng.integers(0, 256, (n, dim), dtype=np.uint8)
    x = rng.standard_normal((n, dim))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def chain_frame(chain: np.ndarray, lead: int, seed: int, total: int | None = None) -> np.ndarray:
    """The chain at rows [lead, lead + len(chain)) of a frame of far rows (TAIL of them after it, or up to `total` rows)."""
    rng = np.random.default_rng(seed)
    n = total if total is not None else lead + len(chain) + TAIL
    f = far_rows(n, chain.shape[1], chain.dtype, rng)
    f[lead:lead + len(chain)] = chain
    return f


def alternation(words: np.ndarray, lead: int, length: int, last_before: int) -> bool:
    """True when chain rows [lead, lead + length) got: a new word at even positions, the previous position's word at odd ones."""
    w = np.asarray(words[lead:lead + length])
    new = w[0::2]
    return bool((new > last_before).all() and len(np.unique(new)) == len(new) and np.array_equal(w[1::2], w[0::2][:len(w[1::2])]))


# ---------------------------------------------------------------------------------------------------------------- ties
def tie_index_vs_new(dim: int, seed: int):
    """(dictionary [1, dim], frame): a one-word dictionary W and a frame whose row 0 is W (one entry in fullResults: a new word X
    equal to W) and whose rows 1, 31, 32, 33, 64 and 95 are W again: the index hit W and the new word X both at distance 0, W wins."""
    rng = np.random.default_rng(seed)
    w = far_rows(1, dim, np.uint8, rng)
    f = far_rows(100, dim, np.uint8, rng)
    f[[0, 1, 31, 32, 33, 64, 95]] = w[0]
    return w, f


TIE_COPIES = (2, 31, 32, 33, 64, 95)


def tie_new_vs_new(dim: int, seed: int) -> np.ndarray:
    """A frame for an EMPTY dictionary: rows 0 and 1 equal x (row 1 sees one entry, so it creates a second word equal to the first);
    x again at TIE_COPIES: both words at distance 0, as chunk-mates (row 2, 31) and as words of an earlier chunk (32 and later); the
    earlier-created word wins.  Two equal words can only be the first two of an empty dictionary, so this is the only way two new
    words tie where the tie decides an id."""
    rng = np.random.default_rng(seed)
    f = far_rows(100, dim, np.uint8, rng)
    f[[0, 1, *TIE_COPIES]] = f[0]
    return f


def tie_index_pair(dim: int, seed: int, n_words: int = 800):
    """(dictionary [n_words, dim], frame): rows 3 and 700 of the dictionary equal; the frame holds copies of them at rows 0, 31, 32
    and 63 among far rows: two index hits at distance 0, the lower row wins."""
    rng = np.random.default_rng(seed)
    d = far_rows(n_words, dim, np.uint8, rng)
    d[700] = d[3]
    f = far_rows(70, dim, np.uint8, rng)
    f[[0, 31, 32, 63]] = d[3]
    return d, f


# ---------------------------------------------------------------------------------------------------------------- NNDR boundary
def nndr_case(best: int, second: int, via: str, dim: int, seed: int, gap: int = 1, n_far: int = 300):
    """(dictionary, frame, query row, row of the best word in the dictionary) with the query R's two nearest candidates at Hamming
    distances best and second.  via "index": both are dictionary words.  via "new": the second is a word X the frame creates `gap`
    rows before R (X's own two index words, 12 bits away, tie, so X is rejected); R's second index hit is then second + 12 away."""
    rng = np.random.default_rng(seed)
    nbits = 8 * dim
    perm = rng.permutation(nbits)
    s1, s2 = perm[:best], perm[best:best + second]
    t1, t2 = perm[best + second:best + second + 12], perm[best + second + 12:best + second + 24]
    r = rng.integers(0, 2, nbits)

    def flip(*sets):
        x = r.copy()
        for s in sets:
            x[s] ^= 1
        return x

    far = far_rows(n_far, dim, np.uint8, rng)
    q = gap + 3
    f = far_rows(q + 5, dim, np.uint8, rng)
    f[q] = _pack(r)
    if via == "index":
        d = np.concatenate([far[:100], _pack(np.stack([flip(s1), flip(s2)])), far[100:]])
    else:
        d = np.concatenate([far[:100], _pack(np.stack([flip(s1), flip(s2, t1), flip(s2, t2)])), far[100:]])
        f[q - gap] = _pack(flip(s2))
    return d, f, q, 100


# ---------------------------------------------------------------------------------------------------------------- frame sizes
FRAME_SIZES = (1, 31, 32, 33, 4095, 4096)


def mixed_frame(vocab: np.ndarray, n: int, seed: int) -> np.ndarray:
    """n descriptors: near copies of dictionary words, near duplicates of each other and random rows."""
    rng = np.random.default_rng(seed)
    dim = vocab.shape[1]
    f = far_rows(n, dim, np.uint8, rng)
    bits = np.unpackbits(vocab[rng.integers(0, len(vocab), n)], axis=1)
    flip = rng.random(bits.shape) < 0.04
    near = rng.random(n) < 0.5
    f[near] = np.packbits(bits ^ flip, axis=1)[near]
    dup = np.flatnonzero(rng.random(n) < 0.15)
    dup = dup[dup > 0]
    src = rng.integers(0, np.maximum(dup, 1))
    sb = np.unpackbits(f[src], axis=1)
    f[dup] = np.packbits(sb ^ (rng.random(sb.shape) < 0.02), axis=1)
    return f


def repeated_frame(dim: int, seed: int, base: int = 64, times: int = 64) -> np.ndarray:
    """base random descriptors, each repeated `times` times, shuffled."""
    rng = np.random.default_rng(seed)
    b = far_rows(base, dim, np.uint8, rng)
    return b[rng.permutation(np.repeat(np.arange(base), times))]
