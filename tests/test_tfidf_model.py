"""The exact model of the GPU TF-IDF likelihood (tests/tfidf_model.py) on the CPU: its idf against decimal arithmetic, its fixed-point
sum on hand-computed cases, and the bound it derives against the reference's float sum — which must hold, and must be sharp enough
to catch a single dropped posting or an nw off by one at bench scale."""
import math
from decimal import Decimal, localcontext

import numpy as np
import pytest

import tfidf_model as tm
from oracle import oracle_py as orc
from rtabmap_b200 import synth


def test_idf_is_the_correctly_rounded_log10_of_the_float_quotient():
    rng = np.random.default_rng(0)
    pairs = [(int(n), int(w)) for n, w in zip(rng.integers(1, 200000, 3000), rng.integers(1, 200050, 3000))]
    pairs += [(n, w) for n in (1, 2, 3, 7, 10, 100, 401, 1000, 10001) for w in (1, 2, 3, n - 1, n, n + 1, 10 * n) if w > 0]
    for n, w in pairs:
        got, amb = tm.idf_gpu(n, [w])
        q = np.float32(n) / np.float32(w)
        with localcontext() as ctx:
            ctx.prec = 40
            exact = Decimal(float(q)).log10() if q != 1 else Decimal(0)
        want = np.float32(float(exact))  # 40 digits, then the nearest double, then the nearest float: no double rounding at this distance
        assert got[0] == want and not amb[0], (n, w)
    assert tm.idf_gpu(0, [1, 5])[0].tolist() == [0.0, 0.0]      # N == 0: nothing (the reference's `if(N)`)
    assert tm.idf_gpu(10, [0])[0].tolist() == [0.0]             # nw == 0
    assert tm.idf_gpu(10, [10])[0].tolist() == [0.0]            # nw == N: log10(1) = 0, the word adds nothing
    assert tm.idf_gpu(10, [20])[0][0] < 0                       # nw > N: negative


def test_libm_log10f_is_within_two_ulps_of_the_gpu_idf():
    """The reference calls log10f; the GPU rounds a double log10.  glibc's log10f is not correctly rounded: it differs from the GPU's idf
    by one ulp in about a quarter of the (N, nw) pairs and by two in a few tenths of a percent (log10f(0.75) is one).  The bound against
    the reference takes the difference each word actually has."""
    n_diff = n_two = n_all = 0
    for n in list(range(1, 400)) + [1000, 4096, 10001, 20000]:
        nw = np.arange(1, n + 51)
        g, amb = tm.idf_gpu(n, nw)
        o = tm.idf_libm(n, nw)
        assert not amb.any()
        d = np.abs(g.astype(np.float64) - o)
        ulp = np.spacing(np.maximum(np.abs(g), np.abs(o))).astype(np.float64)
        assert np.all(d <= 2 * ulp), n
        n_diff += int((g != o).sum())
        n_two += int((d > ulp).sum())
        n_all += len(nw)
    print(f"log10f differs from the GPU idf in {n_diff} of {n_all} (N, nw) pairs, by two ulps in {n_two}")
    assert 0.15 < n_diff / n_all < 0.35


def test_fixed_point_sum_on_hand_computed_cases():
    # word 1 in signatures 1 (twice), 2 and 3; word 2 in signature 1; N = 10: idf(1) = log10(10/3), idf(2) = log10(10/1) = 1
    idx = tm.Index.from_refs({1: {1: 2, 2: 1, 3: 1}, 2: {1: 1}}, {1: 4, 2: 8, 3: 0})
    idf1 = np.float32(math.log10(float(np.float32(10) / np.float32(3))))
    t11 = np.float32(np.float32(2 * idf1) / np.float32(4))
    t21 = np.float32(np.float32(1 * idf1) / np.float32(8))
    fx = lambda t: int(np.rint(float(t) * 2.0 ** 40))
    want = [np.float32((fx(t11) + fx(np.float32(0.25))) * 2.0 ** -40), np.float32(fx(t21) * 2.0 ** -40), 0.0, 0.0, 0.0, 0.0]
    got = tm.gpu_likelihood(idx, [2, 1, 1, 0, -3, 99], [1, 2, 3, 0, -1, 10 ** 6], 10)
    assert got.tolist() == want                                    # ni = 0, ids <= 0 and unknown ids give 0
    assert tm.gpu_likelihood(idx, [1, 2], [1, 2, 3], 0).tolist() == [0, 0, 0]      # N == 0
    assert tm.gpu_likelihood(idx, [0, -1], [1, 2, 3], 10).tolist() == [0, 0, 0]    # no positive id
    # self_ref counts the query signature in nw: word 2 alone with N = 2 then has nw = 2 = N, idf 0
    assert tm.gpu_likelihood(idx, [2], [1], 2, self_ref=1).tolist() == [0.0]
    # the reference's sum equals the model where every idf and every partial sum is exact
    # (N = 1000: word 1 in one signature, idf 3; word 2 in ten, idf 2)
    exact = tm.Index.from_refs({1: {1: 1}, 2: {s: 1 for s in range(1, 11)}}, {s: 2 if s == 2 else 1 for s in range(1, 11)})
    o = tm.oracle_likelihood(exact, [1, 2], [1, 2], 1000)
    assert o.like.tolist() == tm.gpu_likelihood(exact, [1, 2], [1, 2], 1000).tolist() == [5.0, 1.0]


@pytest.fixture(scope="module", params=[1.0, 1.3], ids=["zipf1.0", "zipf1.3"])
def bench_map(request):
    """The bench's map: 49 152 words, 10 000 signatures of 1000 features, Zipf-distributed words (s = 1.3: a few words are in nearly
    every signature)."""
    ids = np.arange(1, 49153, dtype=np.int32)
    m = synth.make_map(ids, 10000, 1000, seed=2, zipf_s=request.param)
    return m, tm.Index.from_csr(m.word_ids, m.row_ptr, m.sig, m.cnt, m.sig_ids, m.ni)


def _query(m, k):
    return m.sig_words[np.random.default_rng(k).integers(0, len(m.sig_ids))]


def test_bound_holds_and_is_sharp_at_bench_scale(bench_map):
    m, idx = bench_map
    n = len(m.sig_ids) + 1
    for k in range(3):
        q = _query(m, k)
        g = tm.gpu_likelihood(idx, q, m.sig_ids, n)
        o = tm.oracle_likelihood(idx, q, m.sig_ids, n)
        assert tm.within_bound(g, o.like, o.bound).all()
        assert np.all(o.sum_running <= o.sum_apriori)
        scored = np.isfinite(o.min_term)
        assert scored.sum() > 9000
        frac = float((o.bound < o.min_term)[scored].mean())
        assert frac >= 0.98, f"the bound exceeds the smallest term in {1 - frac:.2%} of the signatures"
        assert (g != o.like).any()   # the two sums really differ: the bound is doing work


def test_the_cpu_oracle_computes_the_modelled_reference_sum(bench_map):
    m, idx = bench_map
    od = orc.OracleDictionary()
    od.add_words(np.arange(1, 49153, dtype=np.int32), np.zeros((49152, 32), np.uint8))
    od.update()
    od.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    q = _query(m, 7)
    assert np.array_equal(od.likelihood(q, m.sig_ids, len(m.sig_ids) + 1), tm.oracle_likelihood(idx, q, m.sig_ids, len(m.sig_ids) + 1).like)


def test_bound_catches_a_dropped_posting_of_the_longest_list(bench_map):
    """The longest list is the most common word: the smallest idf, the smallest terms.  Dropping any one of its postings (what a
    slice-boundary slip in the kernel's walk would do) must still take the result outside the bound."""
    m, idx = bench_map
    n = len(m.sig_ids) + 1
    q = _query(m, 0)
    words = tm.query_words(q)
    longest = int(words[np.argmax([idx.nw(w) for w in words])])
    o = tm.oracle_likelihood(idx, q, m.sig_ids, n)
    assert tm.within_bound(tm.gpu_likelihood(idx, q, m.sig_ids, n), o.like, o.bound).all()
    sigs = idx.refs(longest)[0]
    for s in np.random.default_rng(1).choice(sigs, 10, replace=False):
        g = tm.gpu_likelihood(idx, q, m.sig_ids, n, skip={(longest, int(s))})
        bad = ~tm.within_bound(g, o.like, o.bound)
        assert bad.tolist() == (m.sig_ids == s).tolist(), f"dropping ({longest}, {s}) is not caught"


@pytest.mark.parametrize("which", ["longest", "median", "shortest"])
@pytest.mark.parametrize("delta", [1, -1])
def test_bound_catches_nw_off_by_one(bench_map, which, delta):
    m, idx = bench_map
    n = len(m.sig_ids) + 1
    q = _query(m, 0)
    words = tm.query_words(q)
    order = np.argsort([idx.nw(w) for w in words], kind="stable")
    w = int(words[{"longest": order[-1], "median": order[len(order) // 2], "shortest": order[0]}[which]])
    o = tm.oracle_likelihood(idx, q, m.sig_ids, n)
    g = tm.gpu_likelihood(idx, q, m.sig_ids, n, nw_offset={w: delta})
    bad = ~tm.within_bound(g, o.like, o.bound)
    holders = np.isin(m.sig_ids, idx.refs(w)[0])
    assert bad[holders].mean() >= 0.99 and not bad[~holders].any(), (w, idx.nw(w), int(bad.sum()))
