"""CPU oracle of rtabmap::BayesFilter — TEST INFRASTRUCTURE ONLY (tests/, smoke(), bench.py CPU legs).

Restates, dense and literal, corelib/src/BayesFilter.cpp:
  computePosterior   :145-270   prior = prediction * lastPosterior; posterior = likelihood .* prior, normalised
  generatePrediction :301-420   one column per place: LC values at the place's graph neighbours (by margin), see addNeighborProb :272-299
  normalize          :437-505   missing neighbour mass onto the diagonal, uniform value for all other places, renormalisation,
                                epsilon cut, virtual-place row
  updatePosterior    :712-737   last posterior re-keyed to the ids of this call (new ids get 0, or 1 for the very first call)
with float (CV_32FC1) storage and the reference's statement order.  The incremental updatePrediction (:507-710,
Bayes/FullPredictionUpdate=false) is the reference's optimisation of the same matrix and is not restated.

Pinning.  The reference holds one vector for this class, archive/2010-LoopClosure/Tests/TestBayesFilter.m (a 10 x 10 table of
floor(1000 * posterior)).  Its prediction matrices come from the 2010 generatePrediction.m, whose pattern format (separate backward /
forward values, no renormalisation) predates the C++ of this tree, so the table pins the RECURSION (computePosterior + updatePosterior:
tests/test_oracle_bayes.py feeds it the 2010 matrices, tests/golden/bayes_golden.json) and NOT generatePrediction / normalize, which
are restated here from BayesFilter.cpp:273-499.  Those two are pinned separately against the reference's own BayesFilter.cpp, compiled
into oracle/_ref/libref_bayes.so (tests/test_oracle_bayes_ref.py).

Two forms of the same filter:
  BayesFilterOracle.prediction / compute_posterior                 dense float matrix, literal; for maps up to a few thousand places
  BayesFilterOracle.sparse_columns / compute_posterior_sparse      no n x n matrix: every column's listed values, its uniform value and
      its scale, computed in float in the reference's statement order (listed sum in ascending neighbour id, then delta, then the
      uniform fill added to the float sum once per filled row, then scale and epsilon cut); the product with the last posterior is
      then taken in float64, as the high-precision reference of the cv::Mat product.  For maps of tens of thousands of places.

The map graph is the caller's (Memory::getNeighborsId, Memory.cpp; graph code is outside the hot path): `neighbors(id)` returns
{neighbour id: margin} for margins 0..len(prediction_lc)-2, the node itself at margin 0.  Ids in `stm` (the short-term memory) are
dropped from every list as generatePrediction does (:338-352).
"""
from __future__ import annotations

import numpy as np

def parse_prediction_lc(text: str) -> list[float]:
    """Bayes/PredictionLC as setPredictionLC reads it (:70-101): space-separated values, each through uStr2Float (a float), kept as
    doubles."""
    return [float(np.float32(float(v))) for v in text.split()]


DEFAULT_PREDICTION_LC = [0.1, 0.36, 0.30, 0.16, 0.062, 0.0151, 0.00255, 0.000324, 2.5e-05, 1.3e-06, 4.8e-08, 1.2e-09, 1.9e-11, 2.2e-13, 1.7e-15,
                         8.5e-18, 2.9e-20, 6.9e-23]  # Parameters.h:363


class BayesFilterOracle:
    def __init__(self, prediction_lc=None, virtual_place_prior: float = 0.9):
        """`prediction_lc`: a Bayes/PredictionLC string (parsed as the reference does, values rounded through float) or a list of
        values used as given."""
        if isinstance(prediction_lc, str):
            prediction_lc = parse_prediction_lc(prediction_lc)
        self.lc = [float(v) for v in (prediction_lc if prediction_lc is not None else DEFAULT_PREDICTION_LC)]
        self.vpp = np.float32(virtual_place_prior)
        f = np.float32
        total = f(0)
        eps = None
        for j, v in enumerate(self.lc):  # setPredictionLC :103-111 (float accumulation of doubles)
            total = f(total + v)
            if j == 0 or v < eps:
                eps = v
        self.total = total
        self.eps = f(eps)
        self.posterior: dict[int, np.float32] = {}

    def reset(self):
        self.posterior = {}

    # ---- generatePrediction + addNeighborProb + normalize (full update) ---------------------------------------------
    def prediction(self, ids, neighbors, stm=()) -> np.ndarray:
        f = np.float32
        n = len(ids)
        P = np.zeros((n, n), np.float32)  # P[row, col]: data[col + row * cols]
        index = {int(i): k for k, i in enumerate(ids) if i > 0}
        vp_used = ids[0] < 0
        done = set()
        for i, pid in enumerate(ids):
            pid = int(pid)
            if pid in done:
                continue
            if pid > 0:
                nb = {k: m for k, m in sorted(neighbors(pid).items()) if k not in stm}
                loop_margin = [k for k, m in nb.items() if m == 0 and k in index]
                assert loop_margin, f"No 0 margin neighbor for signature {pid}"
                for lid in loop_margin:
                    col = index[lid]
                    s = f(0)
                    for k, m in nb.items():
                        if k >= 0 and k in index:
                            v = f(self.lc[m + 1])
                            P[index[k], col] = v
                            s = f(s + v)
                    done.add(lid)
                    self._normalize(P, col, s, vp_used)
            else:
                if self.vpp > 0:
                    if n > 1:
                        P[0, i] = self.vpp
                        P[1:, i] = f((1.0 - float(self.vpp)) / (n - 1))
                    else:
                        P[0, i] = 1
                else:
                    P[:, i] = f(1.0 / n) if n > 1 else f(1)
        return P

    def _normalize(self, P, col, s, vp_used):
        f = np.float32
        n = P.shape[0]
        lc0 = self.lc[0]
        if s < float(self.total) - lc0:
            delta = f(float(self.total) - lc0 - float(s))
            P[col, col] = f(P[col, col] + delta)
            s = f(s + delta)
        other = f(0)
        if self.total < 1:
            other = f(f(1.0) - self.total)
        first = 1 if vp_used else 0
        if other > 0 and n > 1:
            value = f(other / f(n - 1))
            for j in range(first, n):
                if P[j, col] == 0:
                    P[j, col] = value
                    s = f(s + value)
        max_norm = f(1 - (lc0 if vp_used else 0))
        if s < float(max_norm) - 0.0001 or s > float(max_norm) + 0.0001:
            scale = f(max_norm / s)
            for j in range(first, n):
                P[j, col] = f(P[j, col] * scale)
                if P[j, col] < self.eps:
                    P[j, col] = 0
        if vp_used:
            P[0, col] = f(lc0)

    # ---- the same columns without the matrix ---------------------------------------------------------------------------------
    def sparse_columns(self, ids, neighbors, stm=()):
        """Every column of the prediction matrix in sparse form, in float and in the reference's statement order:
        (col_ptr, rows, values, u) where values[e] is P[rows[e], c] for the listed entries of column c and u[c] is the value of every
        other row >= first (first = 1 with a virtual place).  The virtual-place row and column are not included (see _prior)."""
        f = np.float32
        n = len(ids)
        first = 1 if ids[0] < 0 else 0
        col_ptr, rows, levels = prediction_columns(ids, neighbors, stm)
        lcf = np.array([f(v) for v in self.lc], np.float32)
        vals = lcf[levels + 1]
        counts = np.diff(col_ptr)
        real = np.array([i > 0 for i in ids])
        # addNeighborProb: the listed values are added to a float sum in ascending neighbour id
        s = np.zeros(n, np.float32)
        for k in range(int(counts.max(initial=0))):
            c = np.nonzero(counts > k)[0]
            s[c] = (s[c] + vals[col_ptr[c] + k]).astype(np.float32)
        # normalize: the missing mass onto the diagonal (every real column lists its own place)
        entry_col = np.repeat(np.arange(n), counts)
        diag = np.nonzero(rows == entry_col)[0]
        lc0 = self.lc[0]
        need = s.astype(np.float64) < float(self.total) - lc0
        delta = np.zeros(n, np.float32)
        delta[need] = (float(self.total) - lc0 - s[need].astype(np.float64)).astype(np.float32)
        dc = entry_col[diag]
        vals[diag] = np.where(need[dc], (vals[diag] + delta[dc]).astype(np.float32), vals[diag])
        s = np.where(need, (s + delta).astype(np.float32), s)
        # the uniform value of every row still at 0, added to the float sum once per filled row
        other = f(f(1.0) - self.total) if self.total < 1 else f(0)
        value = f(0)
        if other > 0 and n > 1:
            value = f(other / f(n - 1))
            nonzero = np.bincount(entry_col[(vals != 0) & (rows >= first)], minlength=n)
            zeros = (n - first) - nonzero
            s = _repeated_float_add(s, value, np.where(real, zeros, 0))
        # renormalisation and epsilon cut
        max_norm = f(1 - (lc0 if first else 0))
        renorm = real & ((s < float(max_norm) - 0.0001) | (s > float(max_norm) + 0.0001))
        scale = np.where(renorm, (max_norm / np.where(renorm, s, f(1))).astype(np.float32), f(1)).astype(np.float32)
        u = np.where(real, value, f(0)).astype(np.float32)
        vals = np.where(vals == 0, u[entry_col], vals)           # a listed place left at 0 was filled like any other row
        scaled_u = (u * scale).astype(np.float32)
        u = np.where(renorm, np.where(scaled_u < self.eps, f(0), scaled_u), u).astype(np.float32)
        sv = (vals * scale[entry_col]).astype(np.float32)
        rv = renorm[entry_col]
        vals = np.where(rv, np.where(sv < self.eps, f(0), sv), vals).astype(np.float32)
        return col_ptr, rows, vals, u

    def _prior(self, ids, last, col_ptr, rows, vals, u) -> np.ndarray:
        """prior = P x last in float64 from the sparse columns, with the virtual-place row and column of :375-411 / :482-487."""
        n = len(ids)
        vp = ids[0] < 0
        first = 1 if vp else 0
        last64 = last.astype(np.float64)
        entry_col = np.repeat(np.arange(n), np.diff(col_ptr))
        prior = np.zeros(n, np.float64)
        prior[first:] = float(np.dot(u.astype(np.float64), last64))
        np.add.at(prior, rows, (vals.astype(np.float64) - u[entry_col].astype(np.float64)) * last64[entry_col])
        if vp:
            f = np.float32
            if self.vpp > 0:
                p00 = f(self.vpp) if n > 1 else f(1)
                pr0 = f((1.0 - float(self.vpp)) / (n - 1)) if n > 1 else f(0)
            else:
                p00 = pr0 = f(1.0 / n) if n > 1 else f(1)
            prior[0] = float(p00) * last64[0] + float(f(self.lc[0])) * float(last64[1:].sum())
            prior[1:] += float(pr0) * last64[0]
        return prior

    def compute_posterior_sparse(self, ids, likelihood, neighbors, stm=()) -> np.ndarray:
        """computePosterior with the sparse columns and a float64 product; the rest (updatePosterior, the float posterior sum in id
        order, the normalisation) as compute_posterior."""
        ids = [int(i) for i in ids]
        assert ids == sorted(ids), "uKeys(likelihood): ascending ids"
        col_ptr, rows, vals, u = self.sparse_columns(ids, neighbors, stm)
        return self._update(ids, likelihood, lambda last: self._prior(ids, last, col_ptr, rows, vals, u))

    # ---- computePosterior ------------------------------------------------------------------------------------------------
    def compute_posterior(self, ids, likelihood, neighbors=None, prediction=None) -> np.ndarray:
        """`prediction` (dense, float32 [n, n]) overrides generatePrediction — used to replay the reference's 2010 test matrices."""
        ids = [int(i) for i in ids]
        assert ids == sorted(ids), "uKeys(likelihood): ascending ids"
        P = np.asarray(prediction, np.float32) if prediction is not None else self.prediction(ids, neighbors)
        return self._update(ids, likelihood, lambda last: P @ last)  # cv::Mat product, float

    def _update(self, ids, likelihood, product) -> np.ndarray:
        first = len(self.posterior) == 0
        last = np.array([self.posterior.get(i, np.float32(1 if first else 0)) for i in ids], np.float32)  # updatePosterior
        prior = np.asarray(product(last)).astype(np.float32)
        post = (np.asarray(likelihood, np.float32) * prior).astype(np.float32)
        s = np.cumsum(post, dtype=np.float32)[-1]          # float sum in id order (:205-218), one add after the other
        if s != 0:
            post = (post / s).astype(np.float32)
        self.posterior = {i: post[k] for k, i in enumerate(ids)}
        return post


def chain_neighbors(n_levels: int, present=None, loops=None):
    """Neighbour function of a trajectory graph: place k is linked to k-1 and k+1; `loops` adds loop-closure links {a: b} (margin 1
    both ways, as any other link).  BFS by margin, limited to `present` ids when given."""
    loops = loops or {}
    adj_extra: dict[int, set] = {}
    for a, b in loops.items():
        adj_extra.setdefault(a, set()).add(b)
        adj_extra.setdefault(b, set()).add(a)

    def nb(pid: int):
        out = {pid: 0}
        frontier = [pid]
        for m in range(1, n_levels + 1):
            nxt = []
            for u in frontier:
                for v in [u - 1, u + 1, *adj_extra.get(u, ())]:
                    if v >= 1 and v not in out and (present is None or v in present):
                        out[v] = m
                        nxt.append(v)
            frontier = nxt
        return out

    return nb


def graph_tables(places, n_levels: int, links=(), partners=()):
    """{place: {neighbour: margin}} for every place, as Memory::getNeighborsId returns it: a breadth-first walk to margin n_levels over
    `links` (pairs one margin apart) and `partners` (pairs at margin 0: merged places, which share one neighbour tree)."""
    places = [int(p) for p in places]
    adj: dict[int, list] = {p: [] for p in places}
    for a, b in links:
        adj[a].append((b, 1))
        adj[b].append((a, 1))
    for a, b in partners:
        adj[a].append((b, 0))
        adj[b].append((a, 0))
    tables = {}
    for p in places:
        out = {p: 0}
        frontier = [p]
        for m in range(0, n_levels + 1):
            # close the margin-m set over margin-0 links, then step one margin out
            k = 0
            while k < len(frontier):
                for v, w in adj[frontier[k]]:
                    if w == 0 and v not in out:
                        out[v] = m
                        frontier.append(v)
                k += 1
            if m == n_levels:
                break
            nxt = []
            for u in frontier:
                for v, w in adj[u]:
                    if w == 1 and v not in out:
                        out[v] = m + 1
                        nxt.append(v)
            frontier = nxt
        tables[p] = out
    return tables


def _repeated_float_add(s, value, times):
    """s[c] + value + value + ... (times[c] adds), each add rounded to float, as normalize's fill loop does (:457-464).  A literal loop
    over the adds, vectorised across the columns that share a starting sum and an add count."""
    s = np.asarray(s, np.float32)
    times = np.asarray(times, np.int64)
    key = np.stack([s.view(np.int32).astype(np.int64), times], 1)
    uniq, inv = np.unique(key, axis=0, return_inverse=True)
    acc = uniq[:, 0].astype(np.int32).view(np.float32).copy()
    t = uniq[:, 1]
    value = np.float32(value)
    for k in range(int(t.max(initial=0))):
        live = t > k
        acc = np.where(live, acc + value, acc).astype(np.float32)
    return acc[inv.reshape(-1)]


def prediction_columns(ids, neighbors, stm=()):
    """The neighbour lists BayesFilter::generatePrediction ends up using for every column, in CSR form for lcd_bayes_compute_posterior:
    (col_ptr int64 [n+1], nbr_row int32, nbr_level int32).  Same walk as BayesFilterOracle.prediction: places are visited in id order, a
    place and its margin-0 partners (loop-closure links) share the neighbour tree of whichever is visited first (:352-391)."""
    ids = [int(i) for i in ids]
    index = {i: k for k, i in enumerate(ids) if i > 0}
    cols: dict[int, list] = {}
    done = set()
    for pid in ids:
        if pid <= 0 or pid in done:
            continue
        nb = {k: m for k, m in sorted(neighbors(pid).items()) if k not in stm}
        entries = [(index[k], m) for k, m in nb.items() if k >= 0 and k in index]
        for lid in [k for k, m in nb.items() if m == 0 and k in index]:
            cols[index[lid]] = entries
            done.add(lid)
    col_ptr = [0]
    rows, levels = [], []
    for c in range(len(ids)):
        for r, m in cols.get(c, []):
            rows.append(r)
            levels.append(m)
        col_ptr.append(len(rows))
    return np.array(col_ptr, np.int64), np.array(rows, np.int32), np.array(levels, np.int32)
