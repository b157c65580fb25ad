"""Pair matching of the verification step: the tensor-core TO x dictionary scan at its tile edges, and the FROM dictionaries cached
per signature-store row through their life cycle (rows replaced, freed and reused, the store growing, NNDR changing), against the
oracle's RegistrationVis matching and Memory::computeTransform."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth

pytestmark = pytest.mark.gpu

K4 = synth.CAMERA_K4


def random_desc(rng, n, dim):
    return rng.integers(0, 256, (n, dim), dtype=np.uint8)


def run_match(eng, pairs, nndr=0.8):
    cap = max(max(len(f), len(t)) for f, t in pairs)
    cap = max(cap, 1)
    dim = pairs[0][0].shape[1]
    F = np.zeros((len(pairs), cap, dim), np.uint8)
    T = np.zeros((len(pairs), cap, dim), np.uint8)
    for i, (f, t) in enumerate(pairs):
        F[i, :len(f)] = f
        T[i, :len(t)] = t
    fid, tid = eng.match_pairs(F, T, [len(f) for f, _ in pairs], [len(t) for _, t in pairs], nndr)
    for i, (f, t) in enumerate(pairs):
        f_o, t_o = orc.match_pair(f, t, nndr)
        assert np.array_equal(fid[i, :len(f)], f_o), (i, len(f), len(t))
        assert np.array_equal(tid[i, :len(t)], t_o), (i, len(f), len(t))


@pytest.mark.parametrize("dim", [16, 32, 64])
def test_scan_dictionary_and_query_tile_edges(dim):
    """Random FROM descriptors each create a word, so nf is the dictionary size: 0, 1 and both sides of the 8-word, 32-word and
    64-word edges of the scan; TO counts on both sides of the 16-query tile.  Every TO side holds near copies of FROM descriptors
    (accepted matches), exact duplicates of each other (ties) and unrelated descriptors (new words)."""
    rng = np.random.default_rng(dim)
    eng = Engine(desc_dim=dim)
    pairs = []
    for nf, nt in [(0, 5), (1, 1), (1, 17), (7, 16), (8, 15), (9, 33), (31, 32), (32, 31), (33, 48), (63, 64), (64, 65), (65, 63),
                   (127, 129), (128, 128), (129, 127), (300, 301)]:
        f = random_desc(rng, nf, dim)
        t = random_desc(rng, nt, dim)
        if nf:
            src = rng.integers(0, nf, nt)
            near = rng.random(nt) < 0.6
            t[near] = synth.flip_bits(f[src[near]], 0.04, rng)
            t[1::5] = t[0]  # equal distances to every word
        pairs.append((f, t))
    run_match(eng, pairs)
    run_match(eng, pairs, nndr=0.6)


def make_world(dim, n_sig=8, F=300):
    vocab = synth.make_binary_vocabulary(3000, dim, 1)
    ids = np.arange(1, 3001, dtype=np.int32)
    m = synth.make_map(ids, n_sig, F, seed=2)
    st = synth.make_signature_store(vocab, ids, m)
    return m, st


class Fused:
    """lcd_verify_top_dev with a one-hot likelihood: frame b is verified against signature pick[b] of the store."""

    def __init__(self, eng, q, uv, B, F):
        import torch

        self.torch, self.eng, self.B, self.F = torch, eng, B, F
        self.d_q = torch.from_numpy(q.reshape(-1)).cuda()
        self.d_uv = torch.from_numpy(uv.reshape(-1).astype(np.float32)).cuda()

    def run(self, sig_ids, pick, nndr=0.8):
        torch = self.torch
        like = np.zeros((self.B, len(sig_ids)), np.float32)
        col = {int(s): k for k, s in enumerate(sig_ids)}
        for b, h in enumerate(pick):
            like[b, col[int(h)]] = 1.0
        d_l = torch.from_numpy(like.reshape(-1)).cuda()
        d_s = torch.from_numpy(np.asarray(sig_ids, np.int32)).cuda()
        torch.cuda.synchronize()
        self.eng.verify_top_dev(self.d_q.data_ptr(), self.d_uv.data_ptr(), self.B, self.F, d_l.data_ptr(), d_s.data_ptr(), len(sig_ids),
                                Engine.verify_params(K4, nndr=nndr))
        hyp, res = self.eng.process_fetch(self.B)
        assert list(hyp) == [int(h) for h in pick]
        return res


def check(res, rows, q, uv, F, nndr=0.8):
    """rows[b] = (desc, xyz) the store holds for frame b's hypothesis"""
    for b, (desc, xyz) in enumerate(rows):
        v = orc.verify_pair_cov(desc, xyz, q[b * F:(b + 1) * F], uv[b * F:(b + 1) * F], K4, nndr=nndr)
        r = res[b]
        assert r["n_matches"] == len(v["matches"]), (b, r["n_matches"], len(v["matches"]))
        assert r["ok"] == v["ok"] and r["n_inliers"] == len(v["inliers"]), b
        if v["ok"]:
            assert np.allclose(r["rvec"], v["rvec"], atol=1e-4) and np.allclose(r["tvec"], v["tvec"], atol=1e-4)


@pytest.mark.parametrize("dim", [16, 32, 64])
def test_cached_from_dictionaries_follow_the_store(dim):
    m, st = make_world(dim)
    S, F = st.desc.shape[:2]
    B = 6
    q, uv, places, _ = synth.make_query_frames_geo(st, m, B)
    eng = Engine(desc_dim=dim)
    eng.sig_add_batch(m.sig_ids, st.desc, st.xyz)
    fused = Fused(eng, q, uv, B, F)
    row = {int(s): (st.desc[s - 1], st.xyz[s - 1]) for s in m.sig_ids}
    ids = list(m.sig_ids)

    # first use builds, second use reads the cache; duplicate hypotheses in one batch; NNDR 0.8 -> 0.6 -> 0.8
    pick = list(places[:3]) + [places[0]] * 3
    for nndr in (0.8, 0.8, 0.6, 0.8):
        check(fused.run(ids, pick, nndr), [row[int(h)] for h in pick], q, uv, F, nndr)

    # a signature replaced in place with another place's descriptors: the row's cache is stale
    a = int(places[0])
    b = next(int(s) for s in m.sig_ids if s != a)
    eng.sig_add_batch([a], st.desc[b - 1][None], st.xyz[b - 1][None])
    row[a] = row[b]
    check(fused.run(ids, pick), [row[int(h)] for h in pick], q, uv, F)

    # remove, then an add that reuses the freed slot under a new id
    c = int(places[1])
    eng.sig_remove(c)
    ids.remove(c)
    new = S + 1
    d = next(int(s) for s in m.sig_ids if s not in (a, c))
    eng.sig_add_batch([new], st.desc[d - 1][None], st.xyz[d - 1][None])
    assert eng.sig_slots() == S
    ids.append(new)
    row[new] = row[d]
    pick2 = [new if int(h) == c else int(h) for h in pick]
    check(fused.run(ids, pick2), [row[h] for h in pick2], q, uv, F)

    # the store grows (reallocates) after caches were built: they are carried over
    extra = np.arange(S + 2, S + 2 + 3 * S, dtype=np.int32)
    eng.sig_add_batch(extra, np.repeat(st.desc[:1], len(extra), 0), np.repeat(st.xyz[:1], len(extra), 0))
    assert eng.sig_slots() == S + len(extra)
    check(fused.run(ids, pick2), [row[h] for h in pick2], q, uv, F)

    # rows of 0, 1 and 5 descriptors
    small = [S + 10 * S + k for k in range(3)]
    eng.sig_add_batch(small, st.desc[:3], st.xyz[:3], [0, 1, 5])
    ids3 = ids + small
    pick3 = small + small
    rows3 = [(st.desc[k][:n], st.xyz[k][:n]) for k, n in zip(range(3), (0, 1, 5))] * 2
    res = fused.run(ids3, pick3)
    for bi, (desc, xyz) in enumerate(rows3):
        v = orc.verify_pair_cov(desc, xyz, q[bi * F:(bi + 1) * F], uv[bi * F:(bi + 1) * F], K4)
        assert res[bi]["n_matches"] == len(v["matches"]) and res[bi]["ok"] == v["ok"]
