"""The restated loop-closure decision (oracle/decide_py.py) on hand cases for every branch of Rtabmap.cpp:2143-2233 and :3156-3191, and
a multi-step replay of several clients, each with its own compiled reference BayesFilter, over a bayes_cases graph."""
import numpy as np
import pytest

from bayes_cases import PATTERNS, likelihood, make_graph, n_levels, with_vp
from oracle import decide_py as dc
from oracle import oracle_py as orc
from oracle.bayes_py import BayesFilterOracle

IDS = [-1, 3, 5, 8]


def post(*v):
    return np.array(v, np.float32)


def test_ties_go_to_the_highest_id_and_the_value_comes_from_the_virtual_place():
    c = dc.DecideClient(loop_thr=0.11)
    hid, hval, loop, status = c.decide(IDS, post(0.4, 0.2, 0.2, 0.2))
    assert hid == 8 and hval == np.float32(1) - np.float32(0.4) and status == dc.ACCEPTED and loop == 8
    hid, *_ = c.decide(IDS, post(0.1, 0.3, 0.3, 0.3))
    assert hid == 8
    hid, *_ = c.decide(IDS, post(0.1, 0.45, 0.45, 0.0))
    assert hid == 5


def test_no_hypothesis_when_every_real_place_is_zero():
    c = dc.DecideClient()
    hid, hval, loop, status = c.decide(IDS, post(1.0, 0.0, 0.0, 0.0))
    assert (hid, loop, status) == (0, 0, dc.NO_HYPOTHESIS) and hval == 0
    assert c.highest == (0, np.float32(0))


def test_under_threshold_and_the_aggressive_threshold_only_when_lower():
    c = dc.DecideClient(loop_thr=0.11, aggressive_loop_thr=0.05)
    assert c.decide(IDS, post(0.92, 0.02, 0.03, 0.03))[3] == dc.UNDER_THRESHOLD
    assert c.decide(IDS, post(0.92, 0.02, 0.03, 0.03), dc.FRAME_AGGRESSIVE)[3] == dc.ACCEPTED
    c = dc.DecideClient(loop_thr=0.03, aggressive_loop_thr=0.05)   # aggressive higher than LoopThr: not used
    assert c.decide(IDS, post(0.96, 0.01, 0.01, 0.02), dc.FRAME_AGGRESSIVE)[3] == dc.ACCEPTED
    c = dc.DecideClient(loop_thr=0.05, aggressive_loop_thr=0.05)   # equal: LoopThr stays, 0.04 < 0.05
    assert c.decide(IDS, post(0.96, 0.01, 0.01, 0.02), dc.FRAME_AGGRESSIVE)[3] == dc.UNDER_THRESHOLD


def test_single_hypothesis():
    c = dc.DecideClient(loop_thr=0.11)
    assert c.decide([-1, 4], post(0.5, 0.5))[2:] == (0, dc.SINGLE_HYPOTHESIS)
    c = dc.DecideClient(loop_thr=0.0)        # threshold 0: a single hypothesis is accepted
    assert c.decide([-1, 4], post(0.5, 0.5))[2:] == (4, dc.ACCEPTED)


def test_ratio_last_null_and_under_ratio():
    c = dc.DecideClient(loop_thr=0.11, loop_ratio=0.9)
    assert c.decide(IDS, post(0.5, 0.1, 0.3, 0.1))[3] == dc.LAST_NULL            # no last value yet
    assert c.highest == (5, np.float32(0.5))
    assert c.decide(IDS, post(0.6, 0.1, 0.2, 0.1))[3] == dc.RATIO                # 0.4 < 0.9 * 0.5
    assert c.decide(IDS, post(0.62, 0.1, 0.18, 0.1))[3] == dc.ACCEPTED           # 0.38 >= 0.9 * 0.4
    assert c.decide(IDS, post(0.95, 0.01, 0.02, 0.02))[3] == dc.UNDER_RATIO      # 0.05 < thr and < 0.9 * 0.38
    c2 = dc.DecideClient(loop_thr=0.11, loop_ratio=0.0)
    assert c2.decide(IDS, post(0.95, 0.01, 0.02, 0.02))[3] == dc.UNDER_THRESHOLD


def test_skip_and_hold():
    c = dc.DecideClient(loop_thr=0.11, loop_ratio=0.5)
    c.decide(IDS, post(0.3, 0.1, 0.5, 0.1))
    last = c.highest
    assert c.decide(IDS, None, dc.FRAME_HOLD) == (last[0], last[1], 0, dc.HELD) and c.highest == last
    assert c.decide(IDS, None, dc.FRAME_SKIP | dc.FRAME_HOLD) == (0, 0, 0, dc.SKIPPED) and c.highest == (0, 0)
    assert c.decide(IDS, post(0.3, 0.1, 0.5, 0.1))[3] == dc.LAST_NULL             # the skip cleared the last value


def test_verification_and_distance_rejection_leave_the_last_highest_untouched():
    c = dc.DecideClient(loop_thr=0.11, max_loop_closure_distance=2.0)
    d = c.decide(IDS, post(0.3, 0.1, 0.5, 0.1))
    assert d[3] == dc.ACCEPTED
    last = c.highest
    assert c.verified(d, False) == (d[0], d[1], 0, dc.VERIFY_REJECTED) and c.highest == last
    assert c.verified(d, True, (1.5, 1.5, 0.0)) == (d[0], d[1], 0, dc.DISTANCE_REJECTED) and c.highest == last
    assert c.verified(d, True, (1.0, 1.0, 0.5)) == d
    off = dc.DecideClient(loop_thr=0.11, max_loop_closure_distance=0.0)
    d = off.decide(IDS, post(0.3, 0.1, 0.5, 0.1))
    assert off.verified(d, True, (100.0, 0.0, 0.0)) == d
    assert off.verified((5, np.float32(0.2), 0, dc.UNDER_THRESHOLD), False)[3] == dc.UNDER_THRESHOLD


@pytest.mark.parametrize("graph", ["loops", "merged"])
def test_replay_of_several_clients_through_the_reference_filter(graph):
    """Four clients, each with its own compiled BayesFilter.cpp, over ten steps of a growing map: the decisions taken on the reference's
    posterior equal those taken on the sparse restatement's wherever the value is farther than 1e-3 from every threshold, and every
    decision with an accepted hypothesis names the arg-max real place."""
    if orc.ref_bayes_lib() is None:
        pytest.skip("the reference's BayesFilter.cpp is not built")
    text = PATTERNS["default"]
    rng = np.random.default_rng(11)
    n_cl = 4
    refs = [orc.RefBayesFilter(text, 0.9) for _ in range(n_cl)]
    sparse = [BayesFilterOracle(text, 0.9) for _ in range(n_cl)]
    dr = [dc.DecideClient(loop_thr=0.11, loop_ratio=0.5) for _ in range(n_cl)]
    ds = [dc.DecideClient(loop_thr=0.11, loop_ratio=0.5) for _ in range(n_cl)]
    places = list(range(1, 61))
    seen = set()
    for t in range(10):
        places.append(places[-1] + 1)
        ids = with_vp(places, True)
        tables, stm = make_graph(graph, places, n_levels(text), rng)
        for k in range(n_cl):
            flags = dc.FRAME_HOLD if (t + k) % 7 == 3 else (dc.FRAME_AGGRESSIVE if t < 2 else 0)
            like = likelihood(ids, 3 * t + 5 * k, rng)
            if not flags & dc.FRAME_HOLD:
                refs[k].set_graph(tables, stm)
                pr = refs[k].compute_posterior(ids, like)
                ps = sparse[k].compute_posterior_sparse(ids, like, tables.__getitem__, stm)
            else:
                pr = ps = None
            last = float(dr[k].highest[1])
            a = dr[k].decide(ids, pr, flags)
            b = ds[k].decide(ids, ps, flags)
            seen.add(a[3])
            value = a[1]
            near = any(abs(float(value) - float(x)) <= 1e-3 for x in (0.11, 0.05, 0.5 * last))
            if not near:
                assert a[0] == b[0] and a[2:] == b[2:], f"step {t} client {k}"
            if a[3] == dc.ACCEPTED:
                assert a[2] == ids[1 + int(np.argmax(pr[1:]))]
    assert dc.ACCEPTED in seen and dc.HELD in seen
