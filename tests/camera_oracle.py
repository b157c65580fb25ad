"""A camera's local transform (CameraModel::localTransform(), base -> optical) in the oracle's lifting and registration.

Restated from util3d_features.cpp:110-114 (lifting into the base frame, skipped for Transform::isIdentity), util3d_transforms.cpp:211-220
(transformPoint) and util3d_motion_estimation.cpp:154-258 (transform = (localTransform * pnp)^-1, the covariance with
transformCameraFrame = transform * localTransform).  The matching, RANSAC and refinement do not depend on the local transform, so they
are the oracle's own (oracle/oracle_py.py: verify_pair, guess_match, pnp_ransac, match_pair); this module adds what does, in float32
statement by statement, as oracle/oracle_verify.cpp's orcv_covariance computes the identity case.  Transforms are inverted as
[R^T | -R^T t] (the engine's inverse; Eigen's general inverse may differ in the last bits)."""
import math

import numpy as np

from oracle import oracle_py as orc

f32 = np.float32
IDENTITY = np.eye(3, 4, dtype=np.float32)
COV_LINEAR_EPS, COV_ANGULAR_EPS = 0.00000001, 0.00000003   # Registration::COVARIANCE_LINEAR / ANGULAR_EPSILON (Registration.cpp:36-37)


def is_identity(L) -> bool:
    """Transform::isIdentity (Transform.cpp:156-170); None is identity"""
    return L is None or bool(np.array_equal(np.asarray(L, np.float32).reshape(3, 4), IDENTITY))


def transform_point(T, x, y, z):
    """util3d::transformPoint: float32, r0 x + r1 y + r2 z + t, left to right"""
    T = np.asarray(T, np.float32).reshape(3, 4)
    x, y, z = f32(x), f32(y), f32(z)
    return tuple(f32(f32(f32(f32(T[r, 0] * x) + f32(T[r, 1] * y)) + f32(T[r, 2] * z)) + T[r, 3]) for r in range(3))


def lift(xyz, L):
    """generateKeypoints3DDepth's last step: the camera-frame points (NaN = none) into the base frame when L is not identity"""
    xyz = np.asarray(xyz, np.float32)
    if is_identity(L):
        return xyz.copy()
    out = np.full_like(xyz, np.nan)
    for i, p in enumerate(xyz):
        if np.isfinite(p).all():
            out[i] = transform_point(L, *p)
    return out


def tf_mul(A, B):
    """rtabmap::Transform A * B in float: Eigen's 4x4 product with the implicit last row (0 0 0 1), each sum left to right"""
    A, B = np.asarray(A, np.float32).reshape(3, 4), np.asarray(B, np.float32).reshape(3, 4)
    out = np.zeros((3, 4), np.float32)
    for i in range(3):
        for j in range(4):
            v = f32(f32(f32(A[i, 0] * B[0, j]) + f32(A[i, 1] * B[1, j])) + f32(A[i, 2] * B[2, j]))
            out[i, j] = f32(v + A[i, 3]) if j == 3 else v
    return out


def tf_inv(A):
    """[R^T | -R^T t] of a rigid 3x4 float transform"""
    A = np.asarray(A, np.float32).reshape(3, 4)
    out = np.zeros((3, 4), np.float32)
    for i in range(3):
        out[i, :3] = A[:3, i]
        out[i, 3] = -f32(f32(f32(A[0, i] * A[0, 3]) + f32(A[1, i] * A[1, 3])) + f32(A[2, i] * A[2, 3]))
    return out


def pnp_transform(rvec, tvec, L=None):
    """transform = (localTransform * pnp)^-1 of the PnP pose, 3x4 float (util3d_motion_estimation.cpp:145-154)"""
    R = np.zeros(9)
    orc._vlib().orcv_rodrigues(orc._p(np.ascontiguousarray(rvec, np.float64)), orc._p(R))
    P = np.zeros((3, 4), np.float32)
    P[:, :3] = R.reshape(3, 3).astype(np.float32)
    P[:, 3] = np.asarray(tvec, np.float64).astype(np.float32)
    return tf_inv(P if is_identity(L) else tf_mul(L, P))


def covariance(obj, img, obj_to, inliers, T, rvec, tvec, K4, image_size, L=None, var_median_ratio=4, max_variance=0.0, split_linear=False):
    """util3d_motion_estimation.cpp:156-266 for one accepted pose: (accepted, 6x6 covariance before the floor).  obj [n, 3] / img [n, 2]:
    the correspondences given to PnP, obj_to [n, 3] their words3B in the TO base frame (NaN = none) or None, inliers: indices into them."""
    cov = np.eye(6)
    n_inl = len(inliers)
    if n_inl == 0:
        return True, cov
    img_w, img_h = int(image_size[0]), int(image_size[1])
    if obj_to is not None or img_w != 0 or img_h != 0:
        T = np.asarray(T, np.float32).reshape(3, 4)
        C = T.copy() if is_identity(L) else tf_mul(T, L)      # transformCameraFrame
        P = tf_inv(C)                                          # transformCameraFrameInv
        eD, eA, eX, eY, eZ = [], [], [], [], []
        for i in inliers:
            ox, oy, oz = (f32(v) for v in obj[i])
            b = None if obj_to is None else obj_to[i]
            if b is not None and np.isfinite(b).all():
                nx, ny, nz = transform_point(T, *b)
            else:
                zc = transform_point(P, ox, oy, oz)[2]
                fx, fy = f32(K4[0]), f32(K4[1])
                cx, cy = f32(K4[2]), f32(K4[3])
                cx = cx if cx > 0 else f32(f32(img_w // 2) - f32(0.5))
                cy = cy if cy > 0 else f32(f32(img_h // 2) - f32(0.5))
                rx, ry = f32(f32(f32(img[i][0]) - cx) / fx), f32(f32(f32(img[i][1]) - cy) / fy)
                sc = float(zc) * 1.1                            # cv::Point3f * (float * double): per component in double
                nx, ny, nz = transform_point(C, f32(float(rx) * sc), f32(float(ry) * sc), f32(sc))
            dx, dy, dz = f32(ox - nx), f32(oy - ny), f32(oz - nz)
            eD.append(f32(f32(f32(dx * dx) + f32(dy * dy)) + f32(dz * dz)))
            eX.append(f32(float(dx) * float(dx)))
            eY.append(f32(float(dy) * float(dy)))
            eZ.append(f32(float(dz) * float(dz)))
            n1 = np.sqrt(f32(f32(f32(ox * ox) + f32(oz * oz)) + f32(oy * oy)))
            n2 = np.sqrt(f32(f32(f32(nx * nx) + f32(nz * nz)) + f32(ny * ny)))
            ax, ay, az = f32(ox / n1), f32(oy / n1), f32(oz / n1)
            bx, by, bz = f32(nx / n2), f32(ny / n2), f32(nz / n2)
            rad = float(f32(f32(f32(ax * bx) + f32(az * bz)) + f32(ay * by)))
            eA.append(f32(math.acos(min(max(rad, -1.0), 1.0))))
        kth = n_inl // var_median_ratio
        lin = 2.1981 * float(sorted(eD)[kth])
        ang = 2.1981 * float(sorted(eA)[kth])
        for k in range(3):
            cov[k, k] = lin
            cov[k + 3, k + 3] = ang
        if split_linear:
            m = [2.1981 * float(sorted(e)[kth]) for e in (eX, eY, eZ)]
            for k in range(3):
                cov[k, k] = m[k]
            lin = max(m)
        if max_variance > 0 and lin > max_variance:
            return False, np.eye(6)
        return True, cov
    # rms of the inliers' reprojection errors (:253-266): the PnP pose alone, no local transform
    uvp = orc.project_points(np.asarray(obj, np.float32), K4, rvec, tvec)
    err = f32(0)
    for i in inliers:
        ex, ey = f32(f32(img[i][0]) - f32(uvp[i][0])), f32(f32(img[i][1]) - f32(uvp[i][1]))
        err = f32(err + f32(f32(ex * ex) + f32(ey * ey)))
    return True, cov * float(np.sqrt(f32(err / f32(n_inl))))


def _floor(cov):
    for k in range(6):
        eps = COV_LINEAR_EPS if k < 3 else COV_ANGULAR_EPS
        if cov[k, k] <= eps:
            cov[k, k] = eps
    return cov


def register(desc_from, xyz_from, desc_to, uv_to, K4, xyz_to=None, L=None, nndr=0.8, min_inliers=20, iterations=300, reproj=2.0,
             refine_iterations=1, image_size=(640, 480), var_median_ratio=4, max_variance=0.0, split_linear_cov=False, repeat_once=True,
             guess_win_size=40):
    """Memory::computeTransform as oracle_py.verify_pair_repeat computes it, for a TO camera with local transform L (None = identity);
    xyz_to: words3B in the TO base frame.  Returns its dict (matches, inliers, rvec, tvec, transform, covariance, ok, second_pass)."""
    xyz_from = np.asarray(xyz_from, np.float32)
    uv_to = np.asarray(uv_to, np.float32)
    a = orc.verify_pair(desc_from, xyz_from, desc_to, uv_to, K4, nndr=nndr, min_inliers=min_inliers, iterations=iterations, reproj=reproj,
                        refine_iterations=refine_iterations)
    # the correspondences in match order (match ids are the temporary dictionary's word ids)
    fid, tid = orc.match_pair(desc_from, desc_to, nndr)
    f_of = {int(w): i for i, w in enumerate(fid)}
    t_of = {int(w): i for i, w in enumerate(tid)}
    fi = [f_of[int(w)] for w in a["matches"]]
    ti = [t_of[int(w)] for w in a["matches"]]
    pos = {int(w): m for m, w in enumerate(a["matches"])}
    inl = [pos[int(w)] for w in a["inliers"]]
    matches, inliers, rvec, tvec = a["matches"], a["inliers"], a["rvec"], a["tvec"]
    ok, T, cov = False, np.zeros((3, 4), np.float32), np.eye(6)

    def accept(fi, ti, inl, rvec, tvec):
        T = pnp_transform(rvec, tvec, L)
        ok, cov = covariance(xyz_from[fi], uv_to[ti], None if xyz_to is None else np.asarray(xyz_to, np.float32)[ti], inl, T, rvec, tvec, K4,
                             image_size, L, var_median_ratio, max_variance, split_linear_cov)
        return ok, (T if ok else np.zeros((3, 4), np.float32)), cov

    if a["ok"]:
        ok, T, cov = accept(fi, ti, inl, rvec, tvec)
    second = bool(ok and repeat_once and guess_win_size > 0 and image_size[0] > 0 and image_size[1] > 0)
    if second:
        sel, _ = orc.guess_match(desc_from, xyz_from, desc_to, uv_to, K4, rvec, tvec, image_size, guess_win_size, nndr)
        fi = [i for i in range(len(sel)) if sel[i] >= 0]
        ti = [int(sel[i]) for i in fi]
        matches, inliers = np.array(fi, np.int32), np.zeros(0, np.int32)
        ok, T, cov = False, np.zeros((3, 4), np.float32), np.eye(6)
        if len(fi) >= min_inliers:
            _, r, t, idx, _ = orc.pnp_ransac(xyz_from[fi], uv_to[ti], K4, iterations, reproj, min_inliers, refine_iterations, 3.0,
                                             np.concatenate([rvec, tvec]))
            rvec, tvec = r, t
            inliers = matches[idx]
            if len(idx) >= min_inliers:
                ok, T, cov = accept(fi, ti, list(idx), rvec, tvec)
    return {"ok": bool(ok), "matches": np.asarray(matches), "inliers": np.asarray(inliers), "rvec": rvec, "tvec": tvec, "transform": T,
            "covariance": _floor(cov), "second_pass": second}
