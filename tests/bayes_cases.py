"""Inputs shared by the Bayes filter tests (tests/test_oracle_bayes_ref.py on the CPU, tests/test_gpu_bayes_edges.py on the GPU):
Bayes/PredictionLC patterns as a user writes them, and map graphs whose neighbour tables exercise the branches of generatePrediction /
normalize (BayesFilter.cpp:273-499)."""
import numpy as np

from oracle.bayes_py import DEFAULT_PREDICTION_LC, graph_tables

# every pattern is a string, parsed through float as setPredictionLC does
PATTERNS = {
    "default": " ".join(repr(v) for v in DEFAULT_PREDICTION_LC),  # sums to >= 1 in float: no uniform fill
    "sum1": "0.1 0.5 0.2 0.1 0.1",                                # sums to exactly 1
    "trunc5": "0.1 0.36 0.30 0.16 0.062",                         # the default cut to 5 values: uniform fill, epsilon 0.062
    "trunc4": "0.1 0.36 0.30 0.16",
    "largefill": "0.1 0.3 0.1",
    "zerodiag": "0.1 0 0.3 0.1",                                  # margin 0 worth 0: the diagonal becomes non-zero through delta
    "deepzero": "0.1 0.36 0.3 0 0.01",                            # a zero at margin 2: listed places filled like unlisted ones
}
GRAPHS = ("chain", "loops", "merged", "hub", "isolated", "stm")


def n_levels(pattern: str) -> int:
    return len(pattern.split()) - 2


def make_graph(kind: str, places, levels: int, rng):
    """(tables {place: {neighbour: margin}}, stm ids) for a trajectory over `places` (ascending ids):
    chain     consecutive places one margin apart
    loops     the chain plus loop-closure links between distant places
    merged    the chain plus margin-0 partners (merged places share one neighbour tree)
    hub       the chain plus one place linked to up to 320 others
    isolated  the chain with every 7th place unlinked: it lists only itself (all of the pattern's mass goes to delta)
    stm       the chain continued by 5 places of the short-term memory, which are in every table but dropped"""
    places = [int(p) for p in places]
    n = len(places)
    links = [(places[i], places[i + 1]) for i in range(n - 1)]
    partners = []
    stm = []
    if kind == "loops" and n > 8:
        for _ in range(max(1, n // 20)):
            a, b = rng.choice(n, 2, replace=False)
            links.append((places[a], places[b]))
    elif kind == "merged" and n > 4:
        for _ in range(max(1, n // 15)):
            a, b = rng.choice(n, 2, replace=False)
            partners.append((places[a], places[b]))
    elif kind == "hub" and n > 2:
        hub = places[n // 2]
        others = [p for p in places if p != hub]
        for p in rng.choice(others, min(320, len(others)), replace=False):
            links.append((hub, int(p)))
    elif kind == "isolated":
        iso = set(places[::7])
        links = [(a, b) for a, b in links if a not in iso and b not in iso]
    elif kind == "stm":
        stm = list(range(places[-1] + 1, places[-1] + 6))
        links.append((places[-1], stm[0]))
        links += [(stm[i], stm[i + 1]) for i in range(len(stm) - 1)]
    tables = graph_tables(places + stm, levels, links, partners)
    return tables, stm


def with_vp(places, vp: bool):
    return ([-1] if vp else []) + [int(p) for p in places]


def likelihood(ids, t: int, rng):
    """A moving peak over a noisy floor, like Rtabmap::adjustLikelihood's output."""
    like = (1.0 + 0.2 * rng.random(len(ids))).astype(np.float32)
    if len(ids) > 2:
        k = 1 + (5 + 3 * t) % (len(ids) - 1)
        like[k] = 25.0
        like[max(1, k - 1)] = like[min(len(ids) - 1, k + 1)] = 6.0
    return like
