"""The oracle helpers the guess-pass tests build their scenes with: project_points against a plain pinhole projection, and guess_match
(the Reg/RepeatOnce correspondence search, RegistrationVis.cpp:1017-1070, :1225-1370) on scenes small enough to work out by hand."""
import numpy as np

from oracle import oracle_py as orc
from rtabmap_b200 import synth

K4 = (500.0, 500.0, 320.0, 240.0)


def test_project_points_is_the_pinhole_projection():
    rng = np.random.default_rng(3)
    X = np.stack([rng.uniform(-1, 1, 50), rng.uniform(-1, 1, 50), rng.uniform(1, 5, 50)], 1).astype(np.float32)
    rv, tv = np.array([0.05, -0.02, 0.1]), np.array([0.1, -0.2, 0.3])
    c = X.astype(np.float64) @ synth.rodrigues(rv).T + tv
    ref = np.stack([K4[0] * c[:, 0] / c[:, 2] + K4[2], K4[1] * c[:, 1] / c[:, 2] + K4[3]], 1)
    assert np.allclose(orc.project_points(X, K4, rv, tv), ref, rtol=0, atol=1e-9)
    assert np.isnan(orc.project_points(np.full((1, 3), np.nan, np.float32), K4, rv, tv)).all()


def test_guess_match_window_nndr_claims_and_bounds():
    """Identity rotation, zero translation: FROM point (x, y, 1) m projects to (320 + 500 x, 240 + 500 y)."""
    d = np.zeros((6, 32), np.uint8)
    d[:, 0] = np.arange(6) * 16  # distinct rows, far from the 0xFF.. keypoints below
    X = np.array([[0, 0, 1], [0.2, 0, 1], [0.2, 0.02, 1], [-0.4, 0.4, 1], [0, 0, -1], [np.nan, 0, 1]], np.float32)
    # projections: (320, 240), (420, 240), (420, 250), (120, 440), behind the camera, NaN
    dt = np.full((5, 32), 0xFF, np.uint8)
    dt[0] = d[0]
    dt[0, 0] ^= np.uint8(0x0F)  # 4 bits from FROM 0 ...
    dt[1] = d[0]
    dt[1, 0] ^= np.uint8(0x1F)  # ... and 5 bits: 4 < 0.8f * 5 is false
    uv = np.array([[330, 240], [310, 240], [421, 245], [120 + 40, 440], [320, 240]], np.float32)
    sel, n_proj = orc.guess_match(d, X, dt, uv, K4, np.zeros(3), np.zeros(3), image_size=(640, 480), guess_win_size=40, nndr=0.8)
    # FROM 0: candidates 0, 1, 4 (kp 4 at distance 0) -> 3 candidates, best kp 0 (4 bits) vs second kp 1 (5 bits): tie rejected
    # FROM 1 and 2: only kp 2 in their windows -> both select it, the lower index keeps it
    # FROM 3: kp 3 exactly 40 px away -> no candidate; FROM 4 behind the camera; FROM 5 NaN
    assert sel.tolist() == [-1, 2, -1, -1, -1, -1]
    assert n_proj == 4
    # with NNDR 0.9 the 4-vs-5 test passes (4 < 4.5) and FROM 0 takes kp 0
    sel, _ = orc.guess_match(d, X, dt, uv, K4, np.zeros(3), np.zeros(3), image_size=(640, 480), guess_win_size=40, nndr=0.9)
    assert sel.tolist() == [0, 2, -1, -1, -1, -1]
    # a window one pixel wider reaches kp 3
    sel, _ = orc.guess_match(d, X, dt, uv, K4, np.zeros(3), np.zeros(3), image_size=(640, 480), guess_win_size=41, nndr=0.8)
    assert sel[3] == 3
