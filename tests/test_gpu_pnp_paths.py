"""The paths of pnp_ransac_kernel from the RANSAC bookkeeping into the refinement and the covariance: the single-hypothesis path
(n = 6), the Vis/MinInliers gate, no model above 5 inliers, all 300 iterations over three chunks, a refinement that ends below
Vis/MinInliers, the variance rejection, each covariance branch, and a cap other than 1000.  Each case runs through the public
verification calls and is checked against the CPU oracle: inlier lists and iterations_run exact, poses within 1e-7, covariances within
the tolerances of the other verification suites."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine

from test_gpu_verify import K4, make_pair

pytestmark = pytest.mark.gpu

CAP = 700  # a stride other than the benchmark's 1000


def scene(rng, n, outlier_frac=0.3, noise=0.5):
    """n 3-D points and their noisy projections under a small random motion; outlier_frac of them moved anywhere in the image"""
    X = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(0.5, 5, n)], 1).astype(np.float32)
    rv, tv = rng.normal(0, 0.08, 3), rng.normal(0, 0.15, 3)
    import cv2  # only to synthesise the geometry

    K = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1.0]])
    uv, _ = cv2.projectPoints(X.astype(np.float64), rv, tv, K, None)
    uv = (uv.reshape(-1, 2) + rng.normal(0, noise, (n, 2))).astype(np.float32)
    bad = rng.permutation(n)[: int(outlier_frac * n)]
    uv[bad] = np.stack([rng.uniform(0, 640, len(bad)), rng.uniform(0, 480, len(bad))], 1)
    return X, uv


def run_batch(sets, **kw):
    X = np.zeros((len(sets), CAP, 3), np.float32)
    U = np.zeros((len(sets), CAP, 2), np.float32)
    for i, (x, uv) in enumerate(sets):
        X[i, :len(x)], U[i, :len(uv)] = x, uv
    eng = Engine()
    r, t, inl, its = eng.pnp_ransac_batch(X, U, [len(x) for x, _ in sets], K4, **kw)
    eng.close()
    return r, t, inl, its


def assert_pnp_oracle(sets, r, t, inl, its, **kw):
    for i, (x, uv) in enumerate(sets):
        ok, ro, to, io, it = orc.pnp_ransac(x, uv, K4, **kw)
        assert its[i] == it, i
        assert np.array_equal(inl[i], io), i
        assert np.abs(r[i] - ro).max() < 1e-7 and np.abs(t[i] - to).max() < 1e-7, i


def test_ransac_paths_into_the_refinement():
    """n = 6 (one hypothesis), a good scene, and pure outliers: no model above 5 inliers after all 300 iterations (three chunks)"""
    rng = np.random.default_rng(600)
    six = scene(rng, 6, outlier_frac=0.0, noise=0.0)
    good = scene(rng, 500, outlier_frac=0.3)
    junk = (scene(rng, 400)[0], np.stack([rng.uniform(0, 640, 400), rng.uniform(0, 480, 400)], 1).astype(np.float32))
    sets = [six, good, junk, good]
    r, t, inl, its = run_batch(sets, min_inliers=4)
    assert_pnp_oracle(sets, r, t, inl, its, min_inliers=4)
    assert its[0] == 0 and len(inl[0]) == 6  # the single-hypothesis path reports no iterations
    assert its[2] == 300 and len(inl[2]) == 0 and not r[2].any() and not t[2].any()  # best < 0: the guess is kept
    assert 0 < its[1] < 128 and len(inl[1]) >= 300
    assert np.array_equal(inl[1], inl[3]) and its[1] == its[3]


def test_refinement_that_drops_below_min_inliers():
    """RANSAC finds more than Vis/MinInliers inliers; the refinement, whose threshold shrinks to 3 sigma of the errors over five
    passes, keeps fewer: it runs through its "too few new inliers" branch and ends below the minimum"""
    rng = np.random.default_rng(601)
    for _ in range(50):
        x, uv = scene(rng, 60, outlier_frac=0.2, noise=0.7)
        i0 = orc.pnp_ransac(x, uv, K4, min_inliers=4, refine_iterations=0)[3]
        i1 = orc.pnp_ransac(x, uv, K4, min_inliers=4, refine_iterations=5)[3]
        if len(i1) < len(i0):
            break
    else:
        pytest.fail("no scene whose refinement loses inliers")
    kw = {"min_inliers": len(i1) + 1, "refine_iterations": 5}
    sets = [(x, uv)]
    r, t, inl, its = run_batch(sets, **kw)
    assert_pnp_oracle(sets, r, t, inl, its, **kw)
    assert len(inl[0]) < kw["min_inliers"] <= len(i0)


def verify_case(rng, n, cap=CAP, **kw):
    df, x, dt, uv = make_pair(rng, n, outlier_frac=0.3)
    xt = kw.pop("xyz_to", None)
    F = np.zeros((1, cap, 32), np.uint8)
    T = np.zeros((1, cap, 32), np.uint8)
    X = np.full((1, cap, 3), np.nan, np.float32)
    U = np.zeros((1, cap, 2), np.float32)
    F[0, :n], T[0, :n], X[0, :n], U[0, :n] = df, dt, x, uv
    XT = None
    if xt is not None:
        XT = np.full((1, cap, 3), np.nan, np.float32)
        XT[0, :n] = xt(x, dt)
    eng = Engine()
    g = eng.verify_batch(F, X, T, U, K4, [n], [n], xyz_to=XT, **kw)[0]
    eng.close()
    o = orc.verify_pair_cov(df, x, dt, uv, K4, xyz_to=None if XT is None else XT[0, :n], **kw)
    assert g["ok"] == o["ok"]
    assert np.array_equal(g["matches"], o["matches"]) and np.array_equal(g["inliers"], o["inliers"])
    assert np.allclose(g["covariance"], o["covariance"], rtol=1e-4, atol=1e-9)
    if o["ok"]:
        assert np.abs(g["rvec"] - o["rvec"]).max() < 1e-7 and np.abs(g["tvec"] - o["tvec"]).max() < 1e-7
        assert np.allclose(g["transform"], o["transform"], atol=1e-4)
    return g


def words3b(x, dt):
    """3-D points of the TO frame: the FROM points shifted a little, every seventh missing"""
    y = x + np.float32(0.01)
    y[::7] = np.nan
    return y


@pytest.mark.parametrize("branch", ["words3B", "words3B_split", "image_size", "image_size_split", "neither"])
def test_covariance_branches(branch):
    rng = np.random.default_rng(610 + len(branch))
    kw = {"split_linear_cov": branch.endswith("_split")}
    if branch.startswith("words3B"):
        kw["xyz_to"] = words3b
    if branch.startswith("image_size"):
        kw["image_size"] = (640, 480)
    g = verify_case(rng, 600, **kw)
    assert g["ok"] and not np.array_equal(g["covariance"], np.eye(6))


def test_variance_rejection():
    """Vis/PnPMaxVariance below the measured variance: the refined pair is rejected, the covariance goes back to identity"""
    rng = np.random.default_rng(620)
    g = verify_case(rng, 600, image_size=(640, 480), max_variance=1e-9)
    assert not g["ok"] and np.array_equal(g["covariance"], np.eye(6)) and len(g["inliers"]) >= 20


def test_fewer_matches_than_min_inliers():
    """the gate of estimateMotion3DTo2D: PnP does not run, nothing reaches the refinement kernel"""
    rng = np.random.default_rng(630)
    g = verify_case(rng, 15, cap=64, image_size=(640, 480))
    assert not g["ok"] and g["iterations_run"] == 0 and len(g["inliers"]) == 0


def test_mixed_batch_at_another_cap():
    """pairs of every kind side by side at cap 1200, each CTA on its own pair"""
    rng = np.random.default_rng(640)
    cap = 1200
    specs = [(1200, 0.3), (15, 0.0), (700, 0.5), (6, 0.0), (300, 0.2)]
    F = np.zeros((len(specs), cap, 32), np.uint8)
    T = np.zeros((len(specs), cap, 32), np.uint8)
    X = np.full((len(specs), cap, 3), np.nan, np.float32)
    U = np.zeros((len(specs), cap, 2), np.float32)
    raw = []
    for i, (n, of) in enumerate(specs):
        df, x, dt, uv = make_pair(rng, n, outlier_frac=of)
        F[i, :n], T[i, :n], X[i, :n], U[i, :n] = df, dt, x, uv
        raw.append((df, x, dt, uv))
    eng = Engine()
    out = eng.verify_batch(F, X, T, U, K4, [n for n, _ in specs], [n for n, _ in specs], image_size=(640, 480))
    eng.close()
    for i, (df, x, dt, uv) in enumerate(raw):
        o = orc.verify_pair_cov(df, x, dt, uv, K4, image_size=(640, 480))
        g = out[i]
        assert g["ok"] == o["ok"], i
        assert np.array_equal(g["inliers"], o["inliers"]), i
        assert np.allclose(g["covariance"], o["covariance"], rtol=1e-4, atol=1e-9), i
        if o["ok"]:
            assert np.abs(g["rvec"] - o["rvec"]).max() < 1e-7 and np.abs(g["tvec"] - o["tvec"]).max() < 1e-7, i
    assert out[0]["ok"] and not out[1]["ok"] and not out[3]["ok"]
