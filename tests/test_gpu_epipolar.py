"""lcd_epipolar_check_batch (epipolar.cuh) against the CPU restatement of EpipolarGeometry::check (oracle/epipolar_py.py): the pairs of
findPairsUnique, the fundamental-matrix registrators and the check, over the seeded corpus of test_oracle_epipolar.py placed in
signatures with unshared, repeated and negative word ids."""
import numpy as np
import pytest

from epipolar_cases import corpus, point_sets, signature_pair
from oracle import epipolar_py as ep
from rtabmap_b200 import Engine, LcdError
from rtabmap_b200.capi import LCD_DESC_F32

pytestmark = pytest.mark.gpu
CAP = 1200


def _batch(cases):
    n = len(cases)
    ids_a = np.full((n, CAP), -7, np.int32)
    ids_b = np.full((n, CAP), -7, np.int32)
    uv_a = np.zeros((n, CAP, 2), np.float32)
    uv_b = np.zeros((n, CAP, 2), np.float32)
    na = np.zeros(n, np.int32)
    nb = np.zeros(n, np.int32)
    for i, (ia, ua, ib, ub) in enumerate(cases):
        na[i], nb[i] = len(ia), len(ib)
        ids_a[i, :na[i]], uv_a[i, :na[i]] = ia, ua
        ids_b[i, :nb[i]], uv_b[i, :nb[i]] = ib, ub
    return ids_a, uv_a, na, ids_b, uv_b, nb


def _cases(max_n=1000):
    out = []
    for kind, n, o, seed in corpus(max_n):
        p1, p2 = point_sets(n, o, kind, seed)
        out.append(signature_pair(p1, p2, seed + 7, extra=min(n, 60), dup=3, negative=2))
    return out


def _same_up_to_scale(F, G, tol=1e-9):
    if not np.any(F) and not np.any(G):
        return True
    F = F / np.linalg.norm(F)
    G = G / np.linalg.norm(G)
    return min(np.abs(F - G).max(), np.abs(F + G).max()) <= tol


@pytest.fixture(scope="module")
def eng():
    return Engine(device=0)


def _compare(g, st, o, where):
    assert g["checked"] == 1, where
    assert (g["n_pairs"], g["method"], g["found"], g["raised"], g["ok"], g["n_inliers"], g["iterations_run"]) == \
        (o["n_pairs"], o["method"], o["found"], o["raises"], o["ok"], o["n_inliers"], o["iterations"]), where
    if o["found"] and st is not None:
        assert np.array_equal(st[:o["n_pairs"]], o["mask"]), where
        assert _same_up_to_scale(g["F"], o["F"]), where


def test_corpus_against_oracle(eng):
    """Every case of the corpus exactly: pairs, method, found, raised, ok, inliers, iterations, the mask and F to 1e-9.  The kernel and
    the oracle share the fundamental-matrix arithmetic (fm_solver.h) and replay the registrators separately."""
    cases = _cases()
    res, status = eng.epipolar_check_batch(*_batch(cases), with_status=True)
    methods = {}
    for meta, (ia, ua, ib, ub), g, st in zip(corpus(), cases, res, status):
        o = ep.check(ia, ua, ib, ub)
        _compare(g, st, o, meta)
        methods[o["method"]] = methods.get(o["method"], 0) + 1
    print("cases per method:", methods)
    assert methods.get(ep.METHOD_LMEDS, 0) > 100 and methods.get(ep.METHOD_RANSAC, 0) > 300


def test_seven_pairs_against_oracle(eng):
    """VhEp/MatchCountMin 7: seven pairs go through the 7-point kernel alone (mask all ones, the first solution)."""
    cases = _cases(7)
    res, status = eng.epipolar_check_batch(*_batch(cases), match_count_min=7, with_status=True)
    for meta, (ia, ua, ib, ub), g, st in zip(corpus(7), cases, res, status):
        o = ep.check(ia, ua, ib, ub, match_count_min=7)
        assert o["method"] == ep.METHOD_7POINT
        _compare(g, st, o, meta)


def test_batch_position_and_size(eng):
    cases = _cases(300)[::3]
    full = eng.epipolar_check_batch(*_batch(cases))
    rng = np.random.default_rng(3)
    for size in (1, 5, 37, len(cases)):
        pick = rng.choice(len(cases), size, replace=False)
        sub = eng.epipolar_check_batch(*_batch([cases[i] for i in pick]))
        for j, i in enumerate(pick):
            a, b = sub[j], full[i]
            assert {k: v for k, v in a.items() if k != "F"} == {k: v for k, v in b.items() if k != "F"}
            assert np.array_equal(a["F"], b["F"])


def test_params_and_float_engine():
    p1, p2 = point_sets(300, 0.5, "general", 11)
    case = signature_pair(p1, p2, 12, extra=20)
    e = Engine(device=0, desc_type=LCD_DESC_F32, desc_dim=64)
    for mcm, t, c in ((8, 3.0, 0.99), (20, 1.0, 0.999), (8, 0.0, 0.0), (8, -1.0, 1.5)):
        g = e.epipolar_check_batch(*_batch([case]), match_count_min=mcm, ransac_param1=t, ransac_param2=c)[0]
        o = ep.check(*case, match_count_min=mcm, param1=t, param2=c)
        st = e.epipolar_check_batch(*_batch([case]), match_count_min=mcm, ransac_param1=t, ransac_param2=c, with_status=True)[1][0]
        _compare(g, st, o, (mcm, t, c))


def test_errors(eng):
    a = _batch(_cases(7)[:2])
    with pytest.raises(LcdError) as ex:
        big = tuple(np.zeros((2, 4097) + x.shape[2:], x.dtype) if x.ndim > 1 else x for x in a)
        eng.epipolar_check_batch(*big)
    assert ex.value.code == -3
    ids_a, uv_a, na, ids_b, uv_b, nb = a
    for bad_a, bad_b in (([-1, 3], nb), (na, [CAP + 1, 3])):
        with pytest.raises(LcdError) as ex:
            eng.epipolar_check_batch(ids_a, uv_a, np.array(bad_a), ids_b, uv_b, np.array(bad_b))
        assert ex.value.code == -1


def _decision_world(rng):
    from bayes_cases import PATTERNS, make_graph, n_levels, with_vp
    from oracle.bayes_py import parse_prediction_lc, prediction_columns

    places = list(range(1, 41))
    tables, stm = make_graph("chain", places, n_levels(PATTERNS["default"]), rng)
    ids = with_vp(places, True)
    cp, rows, lv = prediction_columns(ids, tables.__getitem__, stm)
    return places, (ids, cp, rows, lv, parse_prediction_lc(PATTERNS["default"]), 0.9)


def test_decision_epipolar():
    """decide, then the check of every frame that reached it (ACCEPTED, RATIO, LAST_NULL) against the word store, for 16 clients over
    two steps: statuses, loop ids and the untouched highest hypotheses equal decide_py's decision with the oracle's check outcome."""
    import torch

    rng = np.random.default_rng(21)
    places, world = _decision_world(rng)
    B, nq, mcm = 16, 400, 60
    for desc in ({}, {"desc_type": LCD_DESC_F32, "desc_dim": 64}):
        e = Engine(device=0, **desc)
        e.clients_create(B)
        e.clients_set_map(*world)
        # each place: 300 words p*1000+k with its first-view keypoints; the store is filled in two batches of different row widths
        views = {p: point_sets(300, 0.2, "general", 5000 + p) for p in places}
        words = {p: (np.arange(300, dtype=np.int32) + 1000 * p) for p in places}
        for batch, cap in ((places[:20], 320), (places[20:], 400)):
            w = np.full((len(batch), cap), -5, np.int32)
            u = np.zeros((len(batch), cap, 2), np.float32)
            for i, p in enumerate(batch):
                w[i, :300], u[i, :300] = words[p], views[p][0]
            e.sig_words_add_batch(batch, w, u, [300] * len(batch))
            if cap == 320:
                # a place added and removed between the batches: the first place of the wider batch takes its freed row while the
                # store widens its rows
                e.sig_words_add_batch([99], np.zeros((1, 8), np.int32), np.zeros((1, 8, 2), np.float32), [8])
                e.sig_words_remove(99)
                assert e.sig_words_count == len(batch)
        assert e.sig_words_count == len(places)
        dp = Engine.decide_params(loop_thr=0.11, loop_ratio=0.9)
        seen = set()
        for t in range(2):
            target = rng.choice(places[:-1], B) if t == 0 else np.array(places[:-1])[rng.choice(39, B)]
            raw = (1.0 + 0.2 * rng.random((B, len(places)))).astype(np.float32)
            peak = np.where(rng.random(B) < 0.7, 40.0, 6.0)
            raw[np.arange(B), target - 1] = peak
            # frame words: the target's words seen from the second view (kind 0), random keypoints (1), or too few shared words (2)
            fw = np.full((B, nq), -3, np.int32)
            fu = np.zeros((B, nq, 2), np.float32)
            fn = np.zeros(B, np.int32)
            for f in range(B):
                p = int(target[f])
                kind = f % 3
                k = 300 if kind != 2 else 40
                perm = rng.permutation(300)[:k]
                fw[f, :k] = words[p][perm]
                fu[f, :k] = views[p][1][perm] if kind != 1 else rng.uniform(0, 640, (k, 2))
                fn[f] = k + 20
                fw[f, k:k + 20] = 900000 + rng.permutation(1000)[:20]
            d_like = torch.from_numpy(raw.reshape(-1)).cuda()
            torch.cuda.synchronize()
            e.decide_batch_dev(d_like.data_ptr(), B, len(places), list(range(B)), [0] * B, dp)
            before = e.decide_fetch(B)
            dw, du, dn = torch.from_numpy(fw).cuda(), torch.from_numpy(fu).cuda(), torch.from_numpy(fn).cuda()
            torch.cuda.synchronize()
            e.decide_epipolar_dev(dw.data_ptr(), du.data_ptr(), dn.data_ptr(), B, nq, match_count_min=mcm)
            after = e.decide_fetch(B)
            res = e.epipolar_fetch(B)
            for f in range(B):
                d0 = tuple(before[f].tolist())
                h = d0[0]
                reached = d0[3] in (dp_status("ratio"), dp_status("last null"), dp_status("accepted"))
                if reached:
                    o = ep.check(fw[f, :fn[f]], fu[f, :fn[f]], words.get(h, np.zeros(0, np.int32)),
                                 views[h][0] if h in views else np.zeros((0, 2), np.float32), match_count_min=mcm)
                    _compare(res[f], None, o, (t, f))
                    expect = ep.decide_epipolar(d0, bool(o["ok"]))
                else:
                    assert res[f]["checked"] == 0
                    expect = d0
                got = tuple(after[f].tolist())
                assert got[0] == expect[0] and got[1] == expect[1] and got[2] == expect[2] and got[3] == expect[3], (t, f, d0, got, expect)
                seen.add(got[3])
        print("statuses seen:", sorted(seen))
        assert ep.EPIPOLAR_REJECTED in seen and dp_status("accepted") in seen and dp_status("last null") in seen


def dp_status(name):
    from rtabmap_b200.capi import DECIDE_STATUS
    return DECIDE_STATUS.index(name)


def test_decision_errors():
    import torch

    e = Engine(device=0)
    d = torch.zeros(64, dtype=torch.int32, device="cuda")
    with pytest.raises(LcdError) as ex:
        e.decide_epipolar_dev(d.data_ptr(), d.data_ptr(), d.data_ptr(), 2, 8)
    assert ex.value.code == -4
    with pytest.raises(LcdError) as ex:
        e.epipolar_fetch(2)
    assert ex.value.code == -4
    rng = np.random.default_rng(3)
    _, world = _decision_world(rng)
    e.clients_create(2)
    e.clients_set_map(*world)
    d_like = torch.ones(2 * 40, dtype=torch.float32, device="cuda")
    e.decide_batch_dev(d_like.data_ptr(), 2, 40, [0, 1], [0, 0], Engine.decide_params())
    for n_frames, nq, code in ((3, 8, -1), (2, 0, -1), (2, 4097, -3)):
        with pytest.raises(LcdError) as ex:
            e.decide_epipolar_dev(d.data_ptr(), d.data_ptr(), d.data_ptr(), n_frames, nq)
        assert ex.value.code == code
    for ids, n, cap, code in (([0], [1], 4, -1), ([5], [5], 4, -1), ([5], [-1], 4, -1), ([5], [1], 4097, -3)):
        with pytest.raises(LcdError) as ex:
            e.sig_words_add_batch(ids, np.zeros((1, cap), np.int32), np.zeros((1, cap, 2), np.float32), n)
        assert ex.value.code == code
    assert e.sig_words_count == 0
