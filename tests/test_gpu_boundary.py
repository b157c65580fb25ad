"""The splice points SURVEY.md §8(b) names, called through the C ABI exactly as the reference's functions are called:
  lcd_pnp_ransac  <-> util3d::solvePnPRansac (util3d_motion_estimation.cpp:843-990), checked against the oracle's restatement and against
                      the OpenCV-derived known answers (tests/golden/pnp_golden.json) WITHOUT going through descriptors;
  lcd_match_bf    <-> cv::BFMatcher::knnMatch / crossCheck match (RegistrationVis.cpp:1128-1141, :1452-1453), checked against cv2 itself
                      (cv::BFMatcher is the third-party implementation the reference calls);
  covariance of util3d::estimateMotion3DTo2D (:156-266) in lcd_verify_result, against the oracle's restatement.
Bit-exact: indices, inlier sets, iteration counts, Hamming distances.  1e-4 (north_star tolerance for float work): poses, covariance."""
import json
import threading
from pathlib import Path

import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import LcdError
from test_gpu_verify import make_pair

pytestmark = pytest.mark.gpu
GOLD = json.loads((Path(__file__).parent / "golden" / "pnp_golden.json").read_text())
K4 = GOLD["K"]


def pnp_problem(rng, n, outliers=0.3, noise=0.5):
    import cv2

    K = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1.0]])
    X = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(0.5, 5, n)], 1).astype(np.float32)
    rv, tv = rng.normal(0, 0.1, 3), rng.normal(0, 0.2, 3)
    uv, _ = cv2.projectPoints(X.astype(np.float64), rv, tv, K, None)
    uv = (uv.reshape(-1, 2) + rng.normal(0, noise, (n, 2))).astype(np.float32)
    bad = rng.permutation(n)[: int(outliers * n)]
    uv[bad] = np.stack([rng.uniform(0, 640, len(bad)), rng.uniform(0, 480, len(bad))], 1)
    return X, uv


@pytest.mark.parametrize("case", GOLD["ransac"], ids=lambda c: f"n{c['n']}_refine{c['refine']}")
def test_pnp_ransac_entry_matches_opencv_golden(case):
    eng = Engine()
    r, t, inl = eng.pnp_ransac(np.asarray(case["X"], np.float32), np.asarray(case["uv"], np.float32), K4, min_inliers=case["min_inliers"],
                               iterations=case["iterations"], reproj_error=case["reproj"], refine_iterations=case["refine"])
    assert inl.tolist() == case["inliers"]
    assert np.allclose(r, case["rvec"], atol=1e-6) and np.allclose(t, case["tvec"], atol=1e-6)


def test_pnp_ransac_entry_matches_oracle():
    rng = np.random.default_rng(5)
    eng = Engine()
    for n, out, refine, min_inl in [(1000, 0.3, 1, 20), (1000, 0.6, 1, 20), (300, 0.5, 0, 20), (40, 0.2, 3, 10), (6, 0.0, 1, 4), (7, 0.0, 1, 4),
                                    (5, 0.0, 1, 4), (25, 0.9, 1, 20)]:
        X, uv = pnp_problem(rng, n, out)
        ok_o, r_o, t_o, inl_o, it_o = orc.pnp_ransac(X, uv, K4, 300, 2.0, min_inl, refine, 3.0, guess=np.zeros(6))
        r, t, inl = eng.pnp_ransac(X, uv, K4, min_inliers=min_inl, refine_iterations=refine)
        assert inl.tolist() == inl_o.tolist(), (n, out)
        if ok_o:
            assert np.allclose(r, r_o, atol=1e-6) and np.allclose(t, t_o, atol=1e-6), (n, out)


def test_pnp_ransac_batch_and_iteration_counts():
    rng = np.random.default_rng(6)
    eng = Engine()
    sizes = [900, 512, 100, 33, 6, 0, 5]
    cap = 900
    X = np.zeros((len(sizes), cap, 3), np.float32)
    uv = np.zeros((len(sizes), cap, 2), np.float32)
    for i, n in enumerate(sizes):
        if n:
            X[i, :n], uv[i, :n] = pnp_problem(rng, n, 0.4)
    r, t, inl, its = eng.pnp_ransac_batch(X, uv, sizes, K4)
    for i, n in enumerate(sizes):
        if n == 0:
            assert len(inl[i]) == 0
            continue
        ok_o, r_o, t_o, inl_o, it_o = orc.pnp_ransac(X[i, :n], uv[i, :n], K4, guess=np.zeros(6))
        assert inl[i].tolist() == inl_o.tolist() and its[i] == it_o
        if ok_o:
            assert np.allclose(r[i], r_o, atol=1e-6) and np.allclose(t[i], t_o, atol=1e-6)


def test_pnp_ransac_no_model_keeps_the_guess_and_rejects_unsupported_input():
    rng = np.random.default_rng(7)
    eng = Engine()
    X, uv = pnp_problem(rng, 5, 0.0)  # fewer than the 6 model points: RANSAC cannot run
    r, t, inl = eng.pnp_ransac(X, uv, K4, rvec=[0.1, 0.2, 0.3], tvec=[1, 2, 3])
    assert len(inl) == 0 and r.tolist() == [0.1, 0.2, 0.3] and t.tolist() == [1, 2, 3]
    X, uv = pnp_problem(rng, 50, 0.1)
    with pytest.raises(LcdError):
        eng.pnp_ransac(X, uv, K4, dist_coeffs=[0.1, 0, 0, 0, 0])
    eng.pnp_ransac(X, uv, K4, dist_coeffs=[0, 0, 0, 0, 0])  # CameraModel::D() of a rectified camera
    with pytest.raises(LcdError):
        eng.pnp_ransac(X, uv, K4, flags=1)
    with pytest.raises(LcdError):
        eng.pnp_ransac(X[:4], uv[:4], K4)


def _cv2_knn(q, t, norm):
    import cv2

    m = cv2.BFMatcher(norm).knnMatch(q, t, k=2)
    i1 = np.array([r[0].trainIdx if len(r) > 0 else -1 for r in m])
    d1 = np.array([r[0].distance if len(r) > 0 else -1 for r in m], np.float32)
    i2 = np.array([r[1].trainIdx if len(r) > 1 else -1 for r in m])
    d2 = np.array([r[1].distance if len(r) > 1 else -1 for r in m], np.float32)
    return i1, d1, i2, d2


def _cv2_cross(q, t, norm):
    import cv2

    out = np.full(len(q), -1)
    dist = np.full(len(q), -1, np.float32)
    for m in cv2.BFMatcher(norm, crossCheck=True).match(q, t):
        out[m.queryIdx] = m.trainIdx
        dist[m.queryIdx] = m.distance
    return out, dist


def test_match_bf_binary_against_cv2():
    import cv2

    rng = np.random.default_rng(8)
    eng = Engine()
    cap = 700
    specs = [(700, 650), (300, 700), (129, 1), (1, 40), (64, 64)]
    Q = np.zeros((len(specs), cap, 32), np.uint8)
    T = np.zeros((len(specs), cap, 32), np.uint8)
    for i, (nq, nt) in enumerate(specs):
        base = rng.integers(0, 256, (max(nq, nt), 32), dtype=np.uint8)
        T[i, :nt] = base[:nt]
        Q[i, :nq] = synth.flip_bits(base[rng.integers(0, nt, nq)], 0.05, rng)
        if nt > 10:
            T[i, 5] = T[i, 3]  # exact duplicates in the train set: ties must go to the lowest index
            T[i, 9] = T[i, 3]
    nq = [s[0] for s in specs]
    nt = [s[1] for s in specs]
    i1, d1, i2, d2 = eng.match_bf(Q, T, nq, nt)
    c1, cd, _, _ = eng.match_bf(Q, T, nq, nt, cross_check=True)
    for i, (a, b) in enumerate(specs):
        o1, od1, o2, od2 = _cv2_knn(Q[i, :a], T[i, :b], cv2.NORM_HAMMING)
        assert np.array_equal(i1[i, :a], o1) and np.array_equal(d1[i, :a], od1)
        assert np.array_equal(i2[i, :a], o2) and np.array_equal(d2[i, :a], od2)
        assert (i1[i, a:] == -1).all()
        oc, ocd = _cv2_cross(Q[i, :a], T[i, :b], cv2.NORM_HAMMING)
        assert np.array_equal(c1[i, :a], oc) and np.array_equal(cd[i, :a], ocd)


def test_match_bf_float_against_cv2():
    import cv2

    rng = np.random.default_rng(9)
    eng = Engine(desc_type=1, desc_dim=64)
    cap = 400
    T = rng.normal(0, 1, (2, cap, 64)).astype(np.float32)
    T /= np.linalg.norm(T, axis=2, keepdims=True)
    Q = (T[:, rng.permutation(cap)] + rng.normal(0, 0.05, T.shape)).astype(np.float32)
    nq, nt = [400, 123], [380, 400]
    i1, d1, i2, d2 = eng.match_bf(Q, T, nq, nt)
    c1, cd, _, _ = eng.match_bf(Q, T, nq, nt, cross_check=True)
    for i in range(2):
        o1, od1, o2, od2 = _cv2_knn(Q[i, :nq[i]], T[i, :nt[i]], cv2.NORM_L2SQR)
        assert np.array_equal(i1[i, :nq[i]], o1) and np.array_equal(i2[i, :nq[i]], o2)
        assert np.allclose(d1[i, :nq[i]], od1, rtol=1e-5) and np.allclose(d2[i, :nq[i]], od2, rtol=1e-5)
        oc, _ = _cv2_cross(Q[i, :nq[i]], T[i, :nt[i]], cv2.NORM_L2SQR)
        assert np.array_equal(c1[i, :nq[i]], oc)


@pytest.mark.parametrize("mode", ["words3B", "ray", "rms", "split", "max_variance"])
def test_verify_covariance_matches_oracle(mode):
    rng = np.random.default_rng(31)
    eng = Engine()
    cap = 600
    pairs = [make_pair(rng, n, outlier_frac=o) for n, o in [(600, 0.3), (300, 0.5), (90, 0.1)]]
    B = len(pairs)
    F = np.zeros((B, cap, 32), np.uint8)
    T = np.zeros((B, cap, 32), np.uint8)
    X = np.full((B, cap, 3), np.nan, np.float32)
    XT = np.full((B, cap, 3), np.nan, np.float32)
    UV = np.zeros((B, cap, 2), np.float32)
    n = []
    for i, (df, x, dt, uv) in enumerate(pairs):
        m = len(df)
        F[i, :m], T[i, :m], X[i, :m], UV[i, :m] = df, dt, x, uv
        # 3-D points of the TO camera: back-projection of its pixels at a plausible depth, a fifth of them missing
        z = rng.uniform(0.5, 5, m).astype(np.float32)
        XT[i, :m] = np.stack([(uv[:, 0] - K4[2]) * z / K4[0], (uv[:, 1] - K4[3]) * z / K4[1], z], 1)
        XT[i, :m:5] = np.nan
        n.append(m)
    kw = dict(var_median_ratio=4)
    xyz_to = None
    if mode in ("words3B", "split", "max_variance"):
        xyz_to = XT
    if mode == "ray":
        kw["image_size"] = (640, 480)
    if mode == "split":
        kw["split_linear_cov"] = True
        kw["var_median_ratio"] = 2
    if mode == "max_variance":
        kw["max_variance"] = 1e-6
    res = eng.verify_batch(F, X, T, UV, K4, n, n, xyz_to=xyz_to, **kw)
    for i in range(B):
        m = n[i]
        o = orc.verify_pair_cov(F[i, :m], X[i, :m], T[i, :m], UV[i, :m], K4, xyz_to=None if xyz_to is None else XT[i, :m], **kw)
        g = res[i]
        assert g["ok"] == o["ok"], (mode, i)
        assert np.array_equal(g["inliers"], o["inliers"])
        assert np.allclose(g["covariance"], o["covariance"], rtol=1e-4, atol=1e-9), (mode, i, np.diag(g["covariance"]), np.diag(o["covariance"]))
        if mode == "max_variance":
            assert not g["ok"] and np.array_equal(g["covariance"], np.eye(6)) and not g["transform"].any()
        elif o["ok"]:
            assert not np.array_equal(g["covariance"], np.eye(6))
            assert np.allclose(g["transform"], o["transform"], atol=1e-4)


def test_signature_store_reuses_freed_rows():
    """One lcd_sig_add + one lcd_sig_remove per frame (the WM -> LTM transfer): the store must not grow (ADVICE r1)."""
    rng = np.random.default_rng(41)
    eng = Engine()
    cap = 50
    d = rng.integers(0, 256, (8, cap, 32), dtype=np.uint8)
    x = rng.normal(0, 1, (8, cap, 3)).astype(np.float32)
    # a refused first add (id 0) stores nothing, so it does not fix the rows per signature either
    with pytest.raises(LcdError) as ex:
        eng.sig_add_batch([0], d[:1, :8], x[:1, :8])
    assert ex.value.code == -1
    assert eng.sig_count() == 0
    eng.sig_add_batch(np.arange(1, 9), d, x)
    assert eng.sig_slots() == 8 and eng.sig_count() == 8
    for k in range(40):
        eng.sig_remove(1 + k)
        eng.sig_add_batch([9 + k], d[k % 8][None], x[k % 8][None])
        assert eng.sig_slots() == 8 and eng.sig_count() == 8
    eng.sig_remove(42)
    eng.sig_remove(45)
    eng.sig_add_batch([100, 101, 102], d[:3], x[:3])  # two freed rows + one fresh
    assert eng.sig_slots() == 9 and eng.sig_count() == 9
    # the reused rows hold the right data: verify signature 101 against itself through the fused call
    vocab = synth.make_binary_vocabulary(256, 32, 1)
    eng.add_words(np.arange(1, 257), vocab)
    eng.update()
    eng.add_refs(101, np.arange(1, 51))
    uv = rng.uniform(0, 400, (1, cap, 2)).astype(np.float32)
    vp = Engine.verify_params(K4, min_inliers=4)
    w, like, hyp, res = eng.process_batch(d[1], uv[0], 1, [101], 2, vp)
    assert res[0]["n_matches"] >= 0  # ran against the stored row of 101 without error


def test_removing_a_word_that_still_has_references_keeps_host_and_device_consistent():
    rng = np.random.default_rng(42)
    eng = Engine()
    o = orc.OracleDictionary()
    vocab = synth.make_binary_vocabulary(64, 32, 3)
    ids = np.arange(1, 65)
    for d in (eng, o):
        d.add_words(ids, vocab)
        d.last_word_id = 64
        d.update()
        d.add_refs(1, [5, 5, 6, 7])
        d.add_refs(2, [5, 8])
    assert eng.total_refs() == 6
    eng.remove_words([5])
    assert eng.total_refs() == 3
    eng.update()
    # word 5 comes back with the same id and gets a new reference; removing signature 1 must not touch it
    eng.add_words([5], vocab[4:5])
    eng.update()
    eng.add_refs(3, [5])
    eng.remove_sig(1)
    sig, cnt = eng.get_refs(5)
    assert sig.tolist() == [3] and cnt.tolist() == [1] and eng.word_nw(5) == 1
    assert eng.total_refs() == 2  # (2, 8) and (3, 5)


def test_orb_detection_runs_beside_dictionary_update():
    """The one concurrency the header allows (Memory.cpp:5284: VWDictionary::update on PreUpdateThread beside feature extraction)."""
    from oracle import feature2d_py as f2d

    eng = Engine(max_words=1 << 17)
    rng = np.random.default_rng(43)
    img = np.stack([synth.make_image(240, 320, 50 + k) for k in range(4)])
    dep = np.stack([synth.make_depth(240, 320, 60 + k) for k in range(4)])
    op = Engine.orb_params(synth.CAMERA_K4, n_features=400)
    ref = eng.orb_detect_describe(img, dep, op)
    words = rng.integers(0, 256, (60000, 32), dtype=np.uint8)
    errors = []

    def updates():
        try:
            nid = 1
            for k in range(30):
                eng.add_words(np.arange(nid, nid + 2000), words[(nid - 1):(nid - 1) + 2000])
                eng.update()
                if k % 3 == 2:
                    eng.remove_words(np.arange(nid, nid + 500))
                nid += 2000
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    t = threading.Thread(target=updates)
    t.start()
    outs = [eng.orb_detect_describe(img, dep, op) for _ in range(12)]
    t.join()
    assert not errors, errors
    for out in outs:
        for (kp, d, x), (kp0, d0, x0) in zip(out, ref):
            assert np.array_equal(kp, kp0) and np.array_equal(d, d0)
    eng.update()  # the rows removed after the last update leave the index now
    assert eng.indexed_size() + eng.not_indexed_size() == eng.size() == 60000 - 10 * 500
    q = words[59000:59010]
    i1, dd1, _, _ = eng.knn2(q)
    assert (dd1 == 0).all()


def test_second_registration_pass_matches_oracle():
    """Reg/RepeatOnce (default true in the reference, Registration.cpp:221-229): after a successful global-matching pass the pair is
    registered again with that transform as the guess — projection of FROM's 3-D points, exact radius search among TO's keypoints,
    knn + strict NNDR among the candidates (RegistrationVis.cpp:1017-1070, :1225-1370).  Correspondence sets and inlier sets exact,
    pose and covariance 1e-4 against the oracle (which, like the kernel, searches the window exactly: see oracle_verify.cpp)."""
    rng = np.random.default_rng(51)
    eng = Engine()
    cap = 800
    specs = [(800, 0.3, 0.04), (500, 0.5, 0.1), (300, 0.1, 0.12), (60, 0.0, 0.02), (25, 0.9, 0.02)]
    pairs = [make_pair(rng, n, flip=f, outlier_frac=o, nan_every=40) for n, o, f in specs]
    B = len(pairs)
    F = np.zeros((B, cap, 32), np.uint8)
    T = np.zeros((B, cap, 32), np.uint8)
    X = np.full((B, cap, 3), np.nan, np.float32)
    UV = np.zeros((B, cap, 2), np.float32)
    n = []
    for i, (df, x, dt, uv) in enumerate(pairs):
        m = len(df)
        F[i, :m], T[i, :m], X[i, :m], UV[i, :m] = df, dt, x, uv
        n.append(m)
    res = eng.verify_batch(F, X, T, UV, K4, n, n, image_size=(640, 480), repeat_once=True, guess_win_size=40)
    res1 = eng.verify_batch(F, X, T, UV, K4, n, n, image_size=(640, 480), repeat_once=False)
    n_second = 0
    for i in range(B):
        m = n[i]
        o = orc.verify_pair_repeat(F[i, :m], X[i, :m], T[i, :m], UV[i, :m], K4, image_size=(640, 480), repeat_once=True, guess_win_size=40)
        g = res[i]
        assert g["ok"] == o["ok"], i
        assert np.array_equal(g["matches"], o["matches"]), i       # ids of the second pass: FROM indices, ascending
        assert np.array_equal(g["inliers"], o["inliers"]), i
        if o["ok"]:
            assert np.allclose(g["rvec"], o["rvec"], atol=1e-4) and np.allclose(g["tvec"], o["tvec"], atol=1e-4)
            assert np.allclose(g["covariance"], o["covariance"], rtol=1e-4, atol=1e-9)
            assert np.allclose(g["transform"], o["transform"], atol=1e-4)
        if o["second_pass"]:
            n_second += 1
            assert not np.array_equal(g["matches"], res1[i]["matches"])   # a different correspondence set than the global matching
        else:
            assert np.array_equal(g["matches"], res1[i]["matches"]) and g["ok"] == res1[i]["ok"]
    assert n_second >= 3
    # without an image size the projection cannot be bounded: the second pass is skipped, as in the reference (isCalibrated = false)
    res0 = eng.verify_batch(F, X, T, UV, K4, n, n, image_size=(0, 0), repeat_once=True)
    for a, b in zip(res0, eng.verify_batch(F, X, T, UV, K4, n, n, image_size=(0, 0), repeat_once=False)):
        assert np.array_equal(a["matches"], b["matches"]) and np.array_equal(a["inliers"], b["inliers"])
