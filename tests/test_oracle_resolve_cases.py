"""The cases of resolve_cases.py produce, on the CPU oracle's sequential new-word loop, the pattern each is built for: without this,
the GPU comparison in test_gpu_resolve_edges.py would not show that the kernel was taken to the edge."""
import numpy as np
import pytest

from oracle import oracle_py as orc
import resolve_cases as rc


def dictionary(words, desc_type=0, nndr=0.8, cmp_new=True):
    o = orc.OracleDictionary(desc_type, words.shape[1], True, nndr, cmp_new)
    if len(words):
        ids = np.arange(1, len(words) + 1, dtype=np.int32)
        o.add_words(ids, words)
        o.last_word_id = len(words)
        o.update()
    return o


@pytest.mark.parametrize("lead", rc.LEADS)
@pytest.mark.parametrize("length,dim", rc.BIN_CHAINS)
def test_binary_chain_alternates(length, dim, lead):
    chain, index = rc.binary_chain(length, dim, seed=length)
    bits = np.unpackbits(chain, axis=1).astype(int)
    d = (bits[:, None] != bits[None]).sum(2)
    assert (np.diag(d, 1) == 4).all() and (d[np.triu_indices(length, 2)] == 8).all()
    ib = np.unpackbits(index, axis=1).astype(int)
    assert ((ib.reshape(length, 2, -1) != bits[:, None]).sum(2) == 9).all()
    o = dictionary(index)
    frame = rc.chain_frame(chain, lead, seed=lead)
    w = o.add_new_words(frame, 1)
    assert rc.alternation(w, lead, length, len(index))
    # without Kp/NewWordsComparedTogether every chain row creates a word
    o2 = dictionary(index, cmp_new=False)
    w2 = o2.add_new_words(frame, 1)
    assert len(np.unique(w2[lead:lead + length])) == length


@pytest.mark.parametrize("lead", rc.LEADS)
@pytest.mark.parametrize("length,dim", rc.F32_CHAINS)
def test_float_chain_alternates(length, dim, lead):
    chain, index = rc.float_chain(length, dim, seed=length)
    o = dictionary(index, desc_type=1)
    w = o.add_new_words(rc.chain_frame(chain, lead, seed=lead), 1)
    assert rc.alternation(w, lead, length, len(index))


@pytest.mark.parametrize("length,dim", rc.BIN_CHAINS)
def test_binary_pair_matching_alternates_the_chain(length, dim):
    """match_pair's FROM pass quantises into an empty dictionary: the planted neighbours first, then the chain"""
    chain, index = rc.binary_chain(length, dim, seed=length)
    src = np.concatenate([index, chain])
    fid, _ = orc.match_pair(src, chain[::-1].copy())
    n_idx_words = len(np.unique(fid[:len(index)]))
    assert rc.alternation(fid, len(index), length, int(fid[:len(index)].max()))
    assert n_idx_words > length


@pytest.mark.parametrize("length,dim", rc.F32_CHAINS)
def test_float_pair_matching_alternates_the_chain(length, dim):
    """The float index words lie along the chain too (all within a few a of each other), so the FROM side is the chain alone: row 0
    creates a word, row 1 sees one entry and creates another, and from there the chain alternates"""
    chain, _ = rc.float_chain(length, dim, seed=length)
    fid, _ = orc.match_pair(chain, chain[::-1].copy())
    assert fid[0] == 1 and rc.alternation(fid, 1, length - 1, 1)


def test_chain_at_the_end_of_a_full_frame():
    length, dim = 100, 32
    chain, index = rc.binary_chain(length, dim, seed=5)
    lead = rc.MAX_FRAME - length
    o = dictionary(index)
    w = o.add_new_words(rc.chain_frame(chain, lead, seed=6, total=rc.MAX_FRAME), 1)
    assert len(w) == rc.MAX_FRAME and rc.alternation(w, lead, length, len(index))


def test_tie_index_word_before_new_word():
    d, f = rc.tie_index_vs_new(32, seed=1)
    o = dictionary(d)
    w = o.add_new_words(f, 1)
    assert w[0] == 2  # one entry in fullResults: a new word equal to the index word
    assert (w[[1, 31, 32, 33, 64, 95]] == 1).all()


def test_tie_earlier_new_word_first_and_one_entry_rule():
    f = rc.tie_new_vs_new(32, seed=2)
    o = dictionary(np.zeros((0, 32), np.uint8))
    w = o.add_new_words(f, 1)
    assert w[0] == 1 and w[1] == 2
    assert (w[list(rc.TIE_COPIES)] == 1).all()


def test_tie_lower_index_row_first():
    d, f = rc.tie_index_pair(32, seed=3)
    o = dictionary(d)
    w = o.add_new_words(f, 1)
    assert (w[[0, 31, 32, 63]] == 4).all()


@pytest.mark.parametrize("gap", [1, 40])
@pytest.mark.parametrize("via", ["index", "new"])
@pytest.mark.parametrize("nndr,best,second,accept", rc.NNDR_CASES)
def test_nndr_boundary(nndr, best, second, accept, via, gap):
    d, f, q, row = rc.nndr_case(best, second, via, 32, seed=best * 100 + second, gap=gap)
    bits = np.unpackbits(d, axis=1).astype(int)
    qb = np.unpackbits(f[q]).astype(int)
    dist = np.sort((bits != qb).sum(1))
    o = dictionary(d, nndr=nndr)
    w = o.add_new_words(f, 1)
    if via == "index":
        assert dist[0] == best and dist[1] == second
    else:
        assert dist[0] == best and dist[1] == second + 12
        x = f[q - gap]
        assert int((np.unpackbits(x).astype(int) != qb).sum()) == second and w[q - gap] > len(d)
    assert (w[q] == row + 1) == accept
    assert accept == (np.float32(best) <= np.float32(nndr) * np.float32(second))
    if (nndr, best, second) == (0.7, 7, 10):
        assert best > float(np.float32(nndr)) * second  # the double product would reject


@pytest.mark.parametrize("n", rc.FRAME_SIZES)
def test_frame_sizes_mix_matches_and_new_words(n):
    rng = np.random.default_rng(n)
    vocab = rng.integers(0, 256, (2000, 32), dtype=np.uint8)
    o = dictionary(vocab)
    w = o.add_new_words(rc.mixed_frame(vocab, n, seed=1000 + n), 1)
    assert len(w) == n
    if n >= 31:
        assert (w <= 2000).any() and (w > 2000).any()
    if n >= 4095:  # rows matched to words created earlier in the frame
        assert len(np.unique(w[w > 2000])) < (w > 2000).sum()


def test_repeated_frame_creates_each_descriptor_once():
    f = rc.repeated_frame(32, seed=4)
    o = dictionary(np.zeros((0, 32), np.uint8))
    w = o.add_new_words(f, 1)
    # only the first row can take the one-entry branch: a word is created twice only when rows 0 and 1 are equal
    assert o.last_word_id == 64 + int(np.array_equal(f[0], f[1]))
    assert len(w) == 4096
