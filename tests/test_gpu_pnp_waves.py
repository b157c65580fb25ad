"""pnp_ransac_kernel solves RANSAC's hypotheses in waves: the EPnP of the first kPnpWave (16) hypotheses, then, only when the run goes
past them, waves of up to kPnpWaveMax (256), so that a 300-iteration run is 16 + 256 + 28.  Each case here ends at or crosses one of
those boundaries and is checked against the CPU oracle at caps 700, 1000 and 1200: iterations_run and the inlier list exact, the pose
within 1e-7, and for the full verification call the covariance within the other suites' tolerance.  The scenes are seeded; the oracle asserts where each run
ends, so a seed that stopped hitting its boundary fails here instead of passing vacuously."""
import ctypes

import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine

from test_gpu_pnp_paths import scene
from test_gpu_verify import K4, make_pair

pytestmark = pytest.mark.gpu

WAVE = 16  # kPnpWave in verify.cuh
N = 600


def samples(n, count):
    """the RANSAC subsets of the first `count` iterations on n points: cv::RNG((uint64)-1) draws, duplicates within a subset redrawn"""
    d = np.zeros(count * 6 + 256, np.uint32)
    orc._vlib().orcv_rng_draws(len(d), n, d.ctypes.data_as(ctypes.c_void_p))
    out, k = [], 0
    for _ in range(count):
        s = []
        while len(s) < 6:
            v = int(d[k])
            k += 1
            if v not in s:
                s.append(v)
        out.append(s)
    return out


def degenerate(x, uv, hyps):
    """the six points of each hypothesis in hyps moved onto one 3-D point: that hypothesis's EPnP returns a non-finite pose"""
    x = x.copy()
    S = samples(len(x), max(hyps) + 1)
    for h in hyps:
        x[S[h]] = x[S[h][0]]
        assert not orc.solve_pnp_epnp(x[S[h]], uv[S[h]], K4)[0]
    return x, uv


def cases():
    """(name, X, uv, check on the oracle's iterations_run)"""
    def sc(seed, of, n=N):
        return scene(np.random.default_rng(seed), n, outlier_frac=of)

    rng = np.random.default_rng(600)
    junk_x = scene(rng, 400)[0]
    junk = (junk_x, np.stack([rng.uniform(0, 640, 400), rng.uniform(0, 480, 400)], 1).astype(np.float32))
    return [
        ("n6", *scene(np.random.default_rng(600), 6, outlier_frac=0.0, noise=0.0), lambda it: it == 0),
        ("inside_wave1", *sc(702, 0.1), lambda it: 0 < it < WAVE),
        ("at_wave_end", *sc(703, 0.2), lambda it: it == WAVE),
        ("one_past_wave", *sc(721, 0.2), lambda it: it == WAVE + 1),
        ("wave2", *sc(705, 0.3), lambda it: WAVE + 1 < it <= 128),
        ("wave3", *sc(748, 0.5), lambda it: 272 < it < 300),
        ("no_model", *junk, lambda it: it == 300),
        ("nonfinite_wave1_and_wave2", *degenerate(*sc(705, 0.3), [3, 40]), lambda it: it > 40),
        ("nonfinite_wave1_only", *degenerate(*sc(702, 0.1), [2]), lambda it: 2 < it < WAVE),
    ]


@pytest.mark.parametrize("cap", [700, 1000, 1200])
def test_pnp_waves_against_oracle(cap):
    cs = cases()
    X = np.zeros((len(cs), cap, 3), np.float32)
    U = np.zeros((len(cs), cap, 2), np.float32)
    for i, (_, x, uv, _) in enumerate(cs):
        X[i, :len(x)], U[i, :len(uv)] = x, uv
    eng = Engine()
    r, t, inl, its = eng.pnp_ransac_batch(X, U, [len(x) for _, x, _, _ in cs], K4, min_inliers=20)
    eng.close()
    for i, (name, x, uv, where) in enumerate(cs):
        ok, ro, to, io, it = orc.pnp_ransac(x, uv, K4, min_inliers=20)
        assert where(it), (name, it)
        assert its[i] == it, (name, its[i], it)
        assert np.array_equal(inl[i], io), name
        assert np.abs(r[i] - ro).max() < 1e-7 and np.abs(t[i] - to).max() < 1e-7, name


@pytest.mark.parametrize("cap", [700, 1000, 1200])
def test_verification_ending_in_each_wave(cap):
    """the full verification call (matching, PnP, refinement, covariance) on pairs whose RANSAC ends in wave 1 and in wave 2"""
    rng = np.random.default_rng(650)
    specs = [(N, 0.05), (N, 0.3), (N, 0.5)]
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
    its = [g["iterations_run"] for g in out]
    assert its[0] <= WAVE < its[1], its
