"""A camera's local transform (CameraModel::localTransform()) in the oracle's lifting and registration (tests/camera_oracle.py): its
identity form is the existing oracle's bit for bit, and a non-identity transform lifts as a literal float32 transformPoint and registers
with the same inliers and errors."""
import numpy as np
import pytest

import camera_oracle as co
from oracle import feature2d_py as f2d
from oracle import oracle_py as orc
from rtabmap_b200 import synth
from rtabmap_b200.capi import OPTICAL_ROTATION, camera_model

K4 = synth.CAMERA_K4
IDENTITY = np.eye(3, 4, dtype=np.float32)


def local(t=(0.3, -0.2, 0.45), yaw=0.2):
    """a base -> optical local transform: a yaw of the base, an offset, then the optical rotation"""
    c, s = np.cos(yaw), np.sin(yaw)
    L = np.eye(4, dtype=np.float32)
    L[:3, :3] = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], np.float32)
    L[:3, 3] = t
    O = np.eye(4, dtype=np.float32)
    O[:3] = OPTICAL_ROTATION
    return (L @ O).astype(np.float32)[:3]


class _Kp:
    def __init__(self, x, y):
        self.pt = (float(x), float(y))


def keypoints(n=400, seed=1):
    rng = np.random.default_rng(seed)
    return [_Kp(x, y) for x, y in zip(rng.uniform(0, 319, n).astype(np.float32), rng.uniform(0, 239, n).astype(np.float32))]


def test_lifting_identity_is_the_plain_restatement():
    depth = synth.make_depth(240, 320, 17)
    a = f2d.keypoints_3d(keypoints(), depth, K4, f2d.OrbParams())
    negzero = IDENTITY.copy()
    negzero[0, 1] = -0.0   # Transform::isIdentity compares values: -0 is 0
    for L in (None, IDENTITY, negzero):
        assert np.array_equal(a.view(np.uint32), co.lift(a, L).view(np.uint32))


def test_lifting_applies_transform_point_in_float32():
    depth = synth.make_depth(240, 320, 17)
    kps = keypoints()
    p = f2d.OrbParams()
    L = local()
    cam = f2d.keypoints_3d(kps, depth, K4, p)
    base = co.lift(cam, L)
    ok = np.isfinite(cam[:, 2])
    assert ok.sum() > 100 and np.array_equal(np.isfinite(base[:, 2]), ok)
    f = np.float32
    for (x, y, z), got in zip(cam[ok], base[ok]):
        want = [f(f(f(f(L[r, 0] * x) + f(L[r, 1] * y)) + f(L[r, 2] * z)) + L[r, 3]) for r in range(3)]
        assert np.array_equal(np.array(want, np.float32).view(np.uint32), got.view(np.uint32))


def test_camera_model_helper():
    c = camera_model(K4, (640, 480), optical=True)
    assert np.array_equal(np.array(c.local_transform[:], np.float32).reshape(3, 4), OPTICAL_ROTATION)
    assert (c.fx, c.fy, c.cx, c.cy, c.image_width, c.image_height) == (*K4, 640, 480)
    L = local()
    c = camera_model(K4, local_transform=L)
    assert np.array_equal(np.array(c.local_transform[:], np.float32).reshape(3, 4), L)


def scene(seed, n=300):
    """a pair observed by camera B with pose (rvec, tvec): FROM 3-D points in A's base frame, TO pixels and TO 3-D points in B's optical frame"""
    rng = np.random.default_rng(seed)
    d_from = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    X = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(1, 5, n)], 1).astype(np.float32)
    rvec, tvec = np.array([0.02, -0.03, 0.01]), np.array([0.1, -0.05, 0.2])
    uv = orc.project_points(X, K4, rvec, tvec).astype(np.float32) + rng.normal(0, 0.3, (n, 2)).astype(np.float32)
    uv[::5] = rng.uniform(0, 300, (len(uv[::5]), 2)).astype(np.float32)
    R = np.zeros(9)
    orc._vlib().orcv_rodrigues(orc._p(np.ascontiguousarray(rvec)), orc._p(R))
    Xb = (X.astype(np.float64) @ R.reshape(3, 3).T + tvec).astype(np.float32)
    Xb[::7] = np.nan
    return d_from, X, synth.flip_bits(d_from, 0.03, rng), uv, Xb


@pytest.mark.parametrize("image_size", [(0, 0), (640, 480)])
@pytest.mark.parametrize("with_3b", [False, True])
@pytest.mark.parametrize("split", [False, True])
def test_identity_registration_is_the_oracle(image_size, with_3b, split):
    """camera_oracle.register with no local transform is oracle_py.verify_pair_repeat bit for bit"""
    d_from, X, d_to, uv, Xb = scene(3)
    kw = dict(xyz_to=Xb if with_3b else None, image_size=image_size, repeat_once=image_size[0] > 0, split_linear_cov=split)
    a = orc.verify_pair_repeat(d_from, X, d_to, uv, K4, **kw)
    b = co.register(d_from, X, d_to, uv, K4, **kw)
    assert a["ok"] and b["ok"] and a["second_pass"] == b["second_pass"]
    for k in ("matches", "inliers", "rvec", "tvec", "transform", "covariance"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    if image_size[0] == 0 and not with_3b:
        return   # the reprojection-RMS covariance has no variance limit
    # a variance limit under the measured one rejects in both
    lim = float(a["covariance"][0, 0]) / 2
    a = orc.verify_pair_repeat(d_from, X, d_to, uv, K4, max_variance=lim, **kw)
    b = co.register(d_from, X, d_to, uv, K4, max_variance=lim, **kw)
    assert not a["ok"] and not b["ok"] and np.array_equal(a["covariance"], b["covariance"])


@pytest.mark.parametrize("image_size", [(0, 0), (640, 480)])
@pytest.mark.parametrize("with_3b", [False, True])
def test_registration_is_invariant_under_the_local_transform(image_size, with_3b):
    """the same correspondences registered with a local transform: the same matches, inliers and PnP pose, a covariance that measures
    the same errors (both are invariant under it) and transform = transform(identity) * localTransform^-1"""
    d_from, X, d_to, uv, Xb = scene(3)
    L = local()
    a = co.register(d_from, X, d_to, uv, K4, xyz_to=Xb if with_3b else None, image_size=image_size, repeat_once=image_size[0] > 0)
    b = co.register(d_from, X, d_to, uv, K4, xyz_to=co.lift(Xb, L) if with_3b else None, image_size=image_size, repeat_once=image_size[0] > 0,
                    L=L)
    assert a["ok"] and b["ok"]
    assert np.array_equal(a["matches"], b["matches"]) and np.array_equal(a["inliers"], b["inliers"])
    assert np.array_equal(a["rvec"], b["rvec"]) and np.array_equal(a["tvec"], b["tvec"])
    np.testing.assert_allclose(b["covariance"], a["covariance"], rtol=1e-3, atol=1e-9)
    L4 = np.eye(4)
    L4[:3] = L
    Ta = np.eye(4)
    Ta[:3] = a["transform"]
    np.testing.assert_allclose(b["transform"], (Ta @ np.linalg.inv(L4))[:3], atol=1e-6)
    # the identity transform given explicitly is the default
    c = co.register(d_from, X, d_to, uv, K4, xyz_to=Xb if with_3b else None, image_size=image_size, repeat_once=image_size[0] > 0, L=IDENTITY)
    assert np.array_equal(c["transform"], a["transform"]) and np.array_equal(c["covariance"], a["covariance"])
