"""An exact model of the GPU TF-IDF likelihood (resolve.cuh score_prep, score.cuh score_kernel<false> + gather_likelihood_kernel), the
reference's own sequential float sum (Memory::computeLikelihood, Memory.cpp:2238-2291), and a bound on how far the two may differ.
Shared by tests/test_tfidf_model.py (CPU) and tests/test_gpu_tfidf_edges.py.

The GPU computes, for every unique query word id w > 0 in ascending order,
    nw  = len(postings of w) + self_ref          (self_ref = 1 in the fused / sharded calls: the query signature counts itself)
    idf = float(log10(double(f32(N) / f32(nw))))  (0 when nw == 0 or N == 0; a word whose idf is 0 adds nothing)
and for every posting (s, nwi) with s > 0 and ni[s] != 0 the float term fl(fl(nwi * idf) / ni[s]), rounded to 2^-40 fixed point
(half to even) and summed in int64 per signature; the output is float(double(acc) * 2^-40).  Every step is reproducible in NumPy, so
the model gives the GPU's bits.  The reference calls log10f instead, and sums the float terms one word after the other."""
from __future__ import annotations

import ctypes
import ctypes.util
from types import SimpleNamespace
from decimal import Decimal, localcontext

import numpy as np

SCALE = 2.0 ** 40
U = 2.0 ** -24  # unit roundoff of float32

_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.log10f.restype = ctypes.c_float
_libm.log10f.argtypes = [ctypes.c_float]


def log10f(x) -> np.float32:
    """The C library's log10f, which the reference (and the CPU oracle) call."""
    return np.float32(_libm.log10f(float(np.float32(x))))


class Index:
    """A mirror of the inverted index: word id -> (signature ids, counts), and ni by signature id."""

    def __init__(self, lists: dict, ni: dict):
        self.lists = {int(w): (np.asarray(s, np.int64), np.asarray(c, np.int64)) for w, (s, c) in lists.items() if len(s)}
        top = max([1] + [int(s.max()) for s, _ in self.lists.values()] + [int(k) for k in ni])
        self.ni = np.zeros(top + 1, np.int64)
        for k, v in ni.items():
            self.ni[int(k)] = int(v)

    @classmethod
    def from_csr(cls, word_ids, row_ptr, sig, cnt, ni_ids, ni_vals):
        rp = np.asarray(row_ptr, np.int64)
        lists = {int(w): (sig[rp[k]:rp[k + 1]], cnt[rp[k]:rp[k + 1]]) for k, w in enumerate(np.asarray(word_ids))}
        return cls(lists, dict(zip(np.asarray(ni_ids).tolist(), np.asarray(ni_vals).tolist())))

    @classmethod
    def from_refs(cls, refs: dict, ni: dict):
        """refs: {word: {signature: count}}"""
        lists = {}
        for w, d in refs.items():
            if d:
                ks = sorted(d)
                lists[w] = (ks, [d[k] for k in ks])
        return cls(lists, ni)

    def refs(self, w: int):
        return self.lists.get(int(w), (np.zeros(0, np.int64), np.zeros(0, np.int64)))

    def nw(self, w: int) -> int:
        return len(self.refs(w)[0])


def query_words(query) -> np.ndarray:
    """uUniqueKeys + the id > 0 test: the unique positive ids, ascending."""
    q = np.unique(np.asarray(query, np.int64))
    return q[q > 0]


def idf_gpu(n_total, nw):
    """(idf [float32], ambiguous [bool]) for arrays of nw: the correctly rounded float of log10(f32(N) / f32(nw)), 0 where nw == 0 or
    N == 0.  `ambiguous` marks the values whose exact logarithm lies so close to a float rounding midpoint that CUDA's double log10
    (1 ulp) could round either way; the model's value there is the correctly rounded one."""
    nw = np.atleast_1d(np.asarray(nw, np.int64))
    out = np.zeros(len(nw), np.float32)
    live = (nw != 0) & (n_total != 0)
    if not live.any():
        return out, np.zeros(len(nw), bool)
    q = (np.float32(n_total) / nw[live].astype(np.float32)).astype(np.float32)
    d = np.log10(q.astype(np.float64))
    f = d.astype(np.float32)
    amb = np.zeros(len(q), bool)
    # the float rounding midpoint nearest to d: between f and its neighbour on d's side
    nb = np.where(d >= f.astype(np.float64), np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf)))
    mid = (f.astype(np.float64) + nb.astype(np.float64)) / 2
    near = np.abs(d - mid) <= 8 * np.spacing(np.abs(d))
    for i in np.flatnonzero(near):
        with localcontext() as ctx:
            ctx.prec = 40
            exact = Decimal(float(q[i])).log10()
            if abs(exact - Decimal(float(nb[i]))) < abs(exact - Decimal(float(f[i]))):
                f[i] = nb[i]
            # CUDA's double log10 is within 1 ulp of the exact value: closer than 2 ulps to the midpoint, it could round either way
            amb[i] = abs(exact - Decimal(float(mid[i]))) <= Decimal(2 * float(np.spacing(abs(d[i]))))
    out[live] = f
    amb_full = np.zeros(len(nw), bool)
    amb_full[live] = amb
    return out, amb_full


def idf_libm(n_total, nw) -> np.ndarray:
    """The reference's idf: log10f(N / nw) on floats (0 where nw == 0 or N == 0)."""
    nw = np.atleast_1d(np.asarray(nw, np.int64))
    out = np.zeros(len(nw), np.float32)
    if n_total == 0:
        return out
    for i, v in enumerate(nw):
        if v:
            out[i] = log10f(np.float32(np.float32(n_total) / np.float32(v)))
    return out


def _terms(index: Index, w: int, idf: np.float32):
    """(signature ids, float32 terms, nwi / ni) of the postings of w that the kernels count: s > 0 and ni[s] != 0."""
    s, c = index.refs(w)  # index.ni covers every posting's signature id
    ni = index.ni[s].astype(np.float32)
    keep = (s > 0) & (ni != 0)
    t = ((c[keep].astype(np.float32) * np.float32(idf)).astype(np.float32) / ni[keep]).astype(np.float32)
    return s[keep], t, c[keep] / ni[keep].astype(np.float64)


def gpu_fixed(index: Index, query, n_total: int, self_ref: int = 0, skip=(), nw_offset=None):
    """The GPU's int64 accumulator by signature id (array of len(index.ni)) and the ambiguous idfs met.
    Mutations for the tests of the bound: skip = {(word, signature)} postings left out, nw_offset = {word: delta}."""
    acc = np.zeros(len(index.ni), np.int64)
    words = query_words(query)
    if n_total == 0 or len(words) == 0:
        return acc, []
    nw = np.array([index.nw(w) + self_ref + (nw_offset or {}).get(int(w), 0) for w in words], np.int64)
    idf, amb = idf_gpu(n_total, nw)
    for w, f in zip(words, idf):
        if f == 0:
            continue
        s, t, _ = _terms(index, w, f)
        fx = np.rint(t.astype(np.float64) * SCALE).astype(np.int64)
        if skip:
            keep = np.array([(int(w), int(x)) not in skip for x in s], bool)
            s, fx = s[keep], fx[keep]
        acc[s] += fx  # a word lists a signature once
    return acc, [(int(n_total), int(v)) for v, a in zip(nw, amb) if a]


def gather(acc: np.ndarray, sig_ids) -> np.ndarray:
    """gather_likelihood_kernel: float(double(acc) * 2^-40) for the listed ids, 0 for ids <= 0 or without an accumulator."""
    s = np.asarray(sig_ids, np.int64)
    ok = (s > 0) & (s < len(acc))
    v = np.zeros(len(s), np.int64)
    v[ok] = acc[s[ok]]
    return (v.astype(np.float64) / SCALE).astype(np.float32)


def gpu_likelihood(index: Index, query, sig_ids, n_total: int, self_ref: int = 0, **mutations) -> np.ndarray:
    acc, amb = gpu_fixed(index, query, n_total, self_ref, **mutations)
    assert not amb, f"idf of (N, nw) {amb[:5]} is within CUDA's log10 error of a float rounding midpoint"
    return gather(acc, sig_ids)


def oracle_likelihood(index: Index, query, sig_ids, n_total: int, self_ref: int = 0):
    """The reference's float sum with log10f, one word after the other in ascending id order, and a bound B on |gpu - oracle| for
    every listed id.  B adds up, over the k terms t_i a signature receives:
      - the idf difference of each term (log10f against the correctly rounded idf: one ulp at least, the actual difference where
        log10f is further off), scaled by nwi / ni, plus the two roundings of each term;
      - the error of the reference's sequential float sum: half an ulp of every partial sum it rounds.  This running form never
        exceeds the a-priori (k - 1) * 2^-24 * sum|t_i| (returned as sum_apriori) and is several times sharper at bench scale;
      - k * 2^-41 of fixed-point rounding on the GPU side;
      - the final rounding of the GPU's double to float (one ulp of the oracle's value covers half an ulp of the GPU's).
    Returns like [float32], bound, min_term (smallest |t_i|, inf where k == 0), sum_running, sum_apriori [float64], by listed id."""
    n = len(index.ni)
    lik = np.zeros(n, np.float32)
    abs_sum = np.zeros(n)
    run_err = np.zeros(n)
    idf_err = np.zeros(n)
    k = np.zeros(n, np.int64)
    tmin = np.full(n, np.inf)
    words = query_words(query)
    if n_total != 0 and len(words):
        nw = np.array([index.nw(w) + self_ref for w in words], np.int64)
        idf_o = idf_libm(n_total, nw)
        idf_g, _ = idf_gpu(n_total, nw)
        for w, fo, fg in zip(words, idf_o, idf_g):
            if fo == 0 and fg == 0:
                continue
            s, t, ratio = _terms(index, w, fo)
            prev = lik[s]
            lik[s] = (prev + t).astype(np.float32)
            run_err[s] += np.where(prev != 0, 0.5 * np.spacing(np.abs(lik[s])).astype(np.float64), 0.0)  # 0 + t is exact
            # glibc's log10f is not correctly rounded: up to 2 ulps from the GPU's idf (0.75 is one such quotient), so the bound takes
            # the difference the two idfs actually have, and one ulp at least
            ulp_idf = max(abs(float(fo) - float(fg)), float(np.spacing(np.float32(max(abs(fo), abs(fg))))))
            at = np.abs(t.astype(np.float64))
            idf_err[s] += ratio * ulp_idf + 2 * np.spacing(np.abs(t)).astype(np.float64)
            abs_sum[s] += at
            k[s] += 1
            tmin[s] = np.minimum(tmin[s], at)
    apriori = np.maximum(k - 1, 0) * U * abs_sum * (1 + 2.0 ** -20)
    bound = idf_err + run_err + k * 2.0 ** -41 + np.spacing(np.abs(lik)).astype(np.float64)
    sid = np.asarray(sig_ids, np.int64)
    ok = (sid > 0) & (sid < n)

    def pick(a, fill):
        v = np.full(len(sid), fill, a.dtype)
        v[ok] = a[sid[ok]]
        return v

    return SimpleNamespace(like=pick(lik, 0), bound=pick(bound, 0), min_term=pick(tmin, np.inf), sum_running=pick(run_err, 0),
                           sum_apriori=pick(apriori, 0))


def within_bound(gpu, oracle, bound) -> np.ndarray:
    return np.abs(np.asarray(gpu, np.float64) - np.asarray(oracle, np.float64)) <= np.asarray(bound)
