"""Reg/RepeatOnce (Registration.cpp:221-229, the reference's default) through the ways a registration reads its pairs: staged host rows
(lcd_verify_batch) and the signature store indexed by hypothesis slot with frame rows of their own stride (the fused query,
lcd_verify_top_dev), at 16, 32 and 64-byte descriptors; the edges of the guess pass on hand-built scenes; and the matching kernel's
size edges (its 1024-thread CTA and the largest cap its shared memory holds).

Two references, as in the rest of the suite: the CPU oracle (verify_pair_repeat, guess_match: correspondence and inlier sets exact,
pose / transform / covariance 1e-4) and lcd_verify_batch on the same pair, bit for bit — the kernels do not depend on where the rows
come from."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import LcdError

pytestmark = pytest.mark.gpu

K4 = synth.CAMERA_K4
IMG = (640, 480)
WIN = 40
DIMS = [16, 32, 64]
LCD_ERR_CAPACITY = -3


# ---------------------------------------------------------------------------------------------------------------- scenes
def make_to(rng, desc, X, rv, tv, nt, flip, outlier_frac, img=IMG):
    """TO side of a view of the FROM points (desc, X) under pose (rv, tv): min(n, nt) keypoints are noisy projections of FROM points
    with flipped descriptor bits (a fraction moved to random pixels), the rest are random keypoints."""
    nf, dim = desc.shape
    m = min(nf, nt)
    uv = orc.project_points(np.nan_to_num(X), K4, rv, tv) + rng.normal(0, 0.5, (nf, 2))
    src = rng.permutation(nf)[:m]
    at = rng.permutation(nt)[:m]
    desc_to = rng.integers(0, 256, (nt, dim), dtype=np.uint8)
    uv_to = np.stack([rng.uniform(0, img[0], nt), rng.uniform(0, img[1], nt)], 1)
    desc_to[at] = synth.flip_bits(desc[src], flip, rng)
    uv_to[at] = uv[src]
    bad = at[rng.random(m) < outlier_frac]
    uv_to[bad] = np.stack([rng.uniform(0, img[0], len(bad)), rng.uniform(0, img[1], len(bad))], 1)
    return desc_to, uv_to.astype(np.float32)


def make_scene(rng, nf, nt, dim, flip=0.06, outlier_frac=0.3, nan_every=40, img=IMG):
    """FROM points back-projected from pixels inside the image at 0.8-6 m under a random pose, and a TO view of them (make_to).
    Returns desc, xyz, desc_to, uv_to, (rv, tv)."""
    rv, tv = rng.normal(0, 0.08, 3), rng.normal(0, 0.15, 3)
    R = synth.rodrigues(rv)
    px = np.stack([rng.uniform(10, img[0] - 10, nf), rng.uniform(10, img[1] - 10, nf)], 1)
    z = rng.uniform(0.8, 6.0, nf)
    cam = np.stack([(px[:, 0] - K4[2]) * z / K4[0], (px[:, 1] - K4[3]) * z / K4[1], z], 1)
    X = ((cam - tv) @ R).astype(np.float32)  # R^T (c - t)
    if nan_every:
        X[::nan_every] = np.nan
    desc = rng.integers(0, 256, (nf, dim), dtype=np.uint8)
    desc_to, uv_to = make_to(rng, desc, X, rv, tv, nt, flip, outlier_frac, img)
    return desc, X, desc_to, uv_to, (rv, tv)


def first_pass_from(desc_from, o1):
    """FROM indices of the correspondences of a global-matching result (its ids are the temporary dictionary's word ids)."""
    fid, _ = orc.match_pair(desc_from, desc_from[:0])
    return sorted(int(np.flatnonzero(fid == w)[0]) for w in o1["matches"])


def second_pass_changed(desc_from, xyz_from, desc_to, uv_to, o2, img=IMG, K=K4):
    """True when the oracle's second pass ran and chose another set of FROM points than its global matching did."""
    if not o2["second_pass"]:
        return False
    o1 = orc.verify_pair_cov(desc_from, xyz_from, desc_to, uv_to, K, image_size=img)
    return first_pass_from(desc_from, o1) != o2["matches"].tolist()


# ---------------------------------------------------------------------------------------------------------------- checks
def assert_oracle(g, o, tag):
    """g: a result of lcd_verify_batch (with "matches" / "inliers") or of the fused calls (counts only)."""
    assert g["ok"] == o["ok"], tag
    if "matches" in g:
        assert np.array_equal(g["matches"], o["matches"]), tag
        assert np.array_equal(g["inliers"], o["inliers"]), tag
    else:
        assert g["n_matches"] == len(o["matches"]) and g["n_inliers"] == len(o["inliers"]), tag
    if o["ok"]:
        assert np.allclose(g["rvec"], o["rvec"], atol=1e-4) and np.allclose(g["tvec"], o["tvec"], atol=1e-4), tag
        assert np.allclose(g["transform"], o["transform"], atol=1e-4), tag
        assert np.allclose(g["covariance"], o["covariance"], rtol=1e-4, atol=1e-9), tag


def assert_same_bits(r, g, tag):
    """r: a fused result, g: lcd_verify_batch's result for the same pair."""
    assert r["ok"] == g["ok"] and r["n_matches"] == len(g["matches"]) and r["n_inliers"] == len(g["inliers"]), tag
    assert r["iterations_run"] == g["iterations_run"], tag
    for k in ("rvec", "tvec", "transform", "covariance"):
        assert r[k].tobytes() == g[k].tobytes(), (tag, k)


def vparams(repeat_once=True, img=IMG, K=K4):
    return Engine.verify_params(K, image_size=img, repeat_once=repeat_once, guess_win_size=WIN)


def batch(eng, rows, frames, cap, dim, repeat_once=True, img=IMG, K=K4, xyz_to=None):
    """lcd_verify_batch of FROM rows[b] = (desc, xyz) against frames[b] = (desc, uv), staged at stride cap"""
    B = len(rows)
    F = np.zeros((B, cap, dim), np.uint8)
    T = np.zeros((B, cap, dim), np.uint8)
    X = np.full((B, cap, 3), np.nan, np.float32)
    U = np.zeros((B, cap, 2), np.float32)
    XT = None if xyz_to is None else np.full((B, cap, 3), np.nan, np.float32)
    for b, ((d, x), (q, uv)) in enumerate(zip(rows, frames)):
        F[b, :len(d)], X[b, :len(d)] = d, x
        T[b, :len(q)], U[b, :len(q)] = q, uv
        if xyz_to is not None:
            XT[b, :len(q)] = xyz_to[b]
    return eng.verify_batch(F, X, T, U, K, [len(d) for d, _ in rows], [len(q) for q, _ in frames], image_size=img, xyz_to=XT,
                            repeat_once=repeat_once, guess_win_size=WIN)


class Fused:
    """lcd_verify_top_dev with one-hot likelihood rows: frame b is registered against signature pick[b] of the store."""

    def __init__(self, eng, frames):
        import torch

        self.torch, self.eng, self.B, self.nq = torch, eng, len(frames), len(frames[0][0])
        q = np.concatenate([f[0] for f in frames])
        uv = np.concatenate([f[1] for f in frames]).astype(np.float32)
        self.d_q = torch.from_numpy(np.ascontiguousarray(q).reshape(-1)).cuda()
        self.d_uv = torch.from_numpy(uv.reshape(-1)).cuda()

    def run(self, sig_ids, pick, vp):
        torch = self.torch
        like = np.zeros((self.B, len(sig_ids)), np.float32)
        col = {int(s): k for k, s in enumerate(sig_ids)}
        for b, h in enumerate(pick):
            like[b, col[int(h)]] = 1.0
        d_l = torch.from_numpy(like.reshape(-1)).cuda()
        d_s = torch.from_numpy(np.asarray(sig_ids, np.int32)).cuda()
        torch.cuda.synchronize()
        self.eng.verify_top_dev(self.d_q.data_ptr(), self.d_uv.data_ptr(), self.B, self.nq, d_l.data_ptr(), d_s.data_ptr(), len(sig_ids), vp)
        hyp, res = self.eng.process_fetch(self.B)
        assert list(hyp) == [int(h) for h in pick]
        return res


# ---------------------------------------------------------------------------------------------------------------- fused query
@pytest.mark.parametrize("st_cap,nq", [(300, 420), (420, 420), (520, 300)], ids=["store_below_nq", "store_equal_nq", "store_above_nq"])
@pytest.mark.parametrize("dim", DIMS)
def test_fused_query_second_pass_matches_oracle_and_verify_batch(dim, st_cap, nq):
    """Store rows through d_hyp_slot (stride st_cap) against frame rows (stride nq), second pass on: duplicate hypotheses, a row with
    fewer descriptors than st_cap, a removed signature (slot -1) and a frame whose first pass fails between two that succeed."""
    rng = np.random.default_rng(1000 + dim + st_cap + nq)
    A = make_scene(rng, st_cap, nq, dim)
    Bs = make_scene(rng, st_cap, nq, dim, flip=0.1, outlier_frac=0.5)
    Cs = make_scene(rng, st_cap, nq, dim, flip=0.12, outlier_frac=0.2)
    n_short = st_cap - 37
    store = {1: (A[0], A[1], st_cap), 2: (Bs[0], Bs[1], n_short), 3: (Cs[0], Cs[1], st_cap), 5: (Cs[0], Cs[1], st_cap)}
    rv, tv = A[4]
    second_view = make_to(rng, A[0], A[1], rv + rng.normal(0, 0.01, 3), tv + rng.normal(0, 0.02, 3), nq, 0.08, 0.4)
    unrelated = (rng.integers(0, 256, (nq, dim), dtype=np.uint8), np.stack([rng.uniform(0, 640, nq), rng.uniform(0, 480, nq)], 1).astype(np.float32))
    frames = [(A[2], A[3]), (Bs[2], Bs[3]), unrelated, (Cs[2], Cs[3]), second_view, (Cs[2], Cs[3])]
    pick = [1, 2, 1, 3, 1, 5]

    eng = Engine(desc_dim=dim)
    ids = sorted(store)
    eng.sig_add_batch(ids, np.stack([store[s][0] for s in ids]), np.stack([store[s][1] for s in ids]), [store[s][2] for s in ids])
    eng.sig_remove(5)  # its hypothesis is still the arg-max of frame 5: no store row (slot -1)
    fused = Fused(eng, frames)
    res = fused.run(ids, pick, vparams())
    res1 = fused.run(ids, pick, vparams(repeat_once=False))

    rows = [(store[h][0][:store[h][2]], store[h][1][:store[h][2]]) if h != 5 else (A[0][:0], A[1][:0]) for h in pick]
    g = batch(eng, rows, frames, max(st_cap, nq), dim)
    changed = 0
    for b, ((d, x), (q, uv)) in enumerate(zip(rows, frames)):
        o = orc.verify_pair_repeat(d, x, q, uv, K4, image_size=IMG, guess_win_size=WIN)
        assert_oracle(g[b], o, ("batch", b))
        assert_oracle(res[b], o, ("fused", b))
        assert_same_bits(res[b], g[b], b)
        if second_pass_changed(d, x, q, uv, o):
            changed += 1
            assert res[b]["n_matches"] != res1[b]["n_matches"] or res[b]["rvec"].tobytes() != res1[b]["rvec"].tobytes(), b
    assert [r["ok"] for r in res] == [True, True, False, True, True, False]
    assert res[5]["n_matches"] == 0
    assert changed >= 3, changed
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- guess-pass edges
def back_project(u, v, z, rv, tv):
    """the world point that projects to pixel (u, v) at camera depth z under (rv, tv); z < 0 puts it behind the camera"""
    R = synth.rodrigues(np.asarray(rv))
    c = np.array([(u - K4[2]) * z / K4[0], (v - K4[3]) * z / K4[1], z])
    return ((c - tv) @ R).astype(np.float32)


def proj32(X, pose):
    return orc.project_points(X[None], K4, *pose)[0].astype(np.float32)


def settle(X, poses, want_x=None):
    """Nudges X[0] by float ulps until both poses project it to the same float pixel (and to x == want_x when given)."""
    for k in range(0, 400):
        for s in (k, -k):
            Y = X.copy()
            Y[0] = np.float32(X[0]) + np.float32(s) * np.spacing(np.float32(X[0]))
            p = [proj32(Y, P) for P in poses]
            if np.array_equal(p[0], p[1]) and (want_x is None or p[0][0] == np.float32(want_x)):
                return Y, p[0]
    raise AssertionError("no float point projects identically under both poses")


@pytest.mark.parametrize("dim", DIMS)
def test_guess_pass_edges_match_oracle(dim):
    """FROM points with unique descriptors, each with a NaN-depth twin of the same descriptor (so its word is not unique and the global
    matching, hence the first pass and its pose, is unchanged), projected into an empty part of a 1280 x 960 image under the first
    pass's pose; TO keypoints placed relative to those projections.  Expected selections are the oracle's, pinned per edge."""
    img = (1280, 960)
    rng = np.random.default_rng(70 + dim)
    d0, x0, dt0, uv0, _ = make_scene(rng, 300, 300, dim, flip=0.04, outlier_frac=0.2, nan_every=0, img=(640, 480))
    eng = Engine(desc_dim=dim)
    o1 = orc.verify_pair_cov(d0, x0, dt0, uv0, K4, image_size=img)
    g1 = batch(eng, [(d0, x0)], [(dt0, uv0)], 300, dim, repeat_once=False, img=img)[0]
    assert o1["ok"] and g1["ok"]
    poses = [(o1["rvec"], o1["tvec"]), (g1["rvec"], g1["tvec"])]  # the guesses of the oracle and of the kernel

    from_d, from_x, to_d, to_uv, expect = [], [], [], [], {}

    def rand_desc():
        return rng.integers(0, 256, (1, dim), dtype=np.uint8)

    def near(desc, nbits):
        out = desc.copy()
        for b in rng.choice(dim * 8, nbits, replace=False):
            out[0, b // 8] ^= np.uint8(1 << (b % 8))
        return out

    def add_from(X, desc, name):
        expect[name] = [300 + len(from_d), None]
        from_d.append(desc)
        from_x.append(X)
        return expect[name]

    def add_to(desc, u, v):
        to_d.append(desc)
        to_uv.append(np.array([u, v], np.float32))
        return 300 + len(to_d) - 1

    # exactly one candidate, far in descriptor space: accepted without the NNDR test
    X, p = settle(back_project(760, 600, 3.0, *poses[0]), poses)
    e = add_from(X, rand_desc(), "single")
    e[1] = add_to(rand_desc(), p[0] + 25, p[1] + 10)
    # a keypoint exactly win pixels away (squared distance == win^2) is no candidate; one float below it is
    X, p = settle(back_project(860, 600, 3.0, *poses[0]), poses)
    add_from(X, rand_desc(), "at_win")
    add_to(rand_desc(), p[0] + np.float32(WIN), p[1])
    X, p = settle(back_project(860, 700, 3.0, *poses[0]), poses)
    e = add_from(X, rand_desc(), "inside_win")
    e[1] = add_to(rand_desc(), np.nextafter(p[0] + np.float32(WIN), np.float32(0)), p[1])
    # d1 == nndr * d2 (4 vs 5 bits: 0.8f * 5 rounds to 4.0f) fails the strict test; 4 vs 6 passes
    X, p = settle(back_project(960, 600, 3.0, *poses[0]), poses)
    dq = rand_desc()
    add_from(X, dq, "nndr_tie")
    add_to(near(dq, 4), p[0] + 5, p[1] + 5)
    add_to(near(dq, 5), p[0] - 5, p[1] - 5)
    X, p = settle(back_project(960, 700, 3.0, *poses[0]), poses)
    dq = rand_desc()
    e = add_from(X, dq, "nndr_pass")
    e[1] = add_to(near(dq, 4), p[0] + 5, p[1] + 5)
    add_to(near(dq, 6), p[0] - 5, p[1] - 5)
    # two FROM points whose only candidate is one keypoint: the lower FROM index takes it, although the higher one is closer in descriptor
    Xa, pa = settle(back_project(1060, 600, 3.0, *poses[0]), poses)
    Xb, pb = settle(back_project(1060, 612, 3.0, *poses[0]), poses)
    db = rand_desc()
    ea = add_from(Xa, rand_desc(), "claim_low")
    add_from(Xb, db, "claim_high")
    ea[1] = add_to(near(db, 2), pa[0] + 4, pa[1] + 6)
    # projection at x == w - 1 (out: the bound is strict) and just below it (in)
    X, p = settle(back_project(img[0] - 1, 800, 3.0, *poses[0]), poses, want_x=img[0] - 1)
    add_from(X, rand_desc(), "x_w_minus_1")
    add_to(rand_desc(), img[0] - 10, p[1])
    X, p = settle(back_project(img[0] - 1.01, 880, 3.0, *poses[0]), poses)
    assert p[0] < img[0] - 1
    e = add_from(X, rand_desc(), "x_below_w_minus_1")
    e[1] = add_to(rand_desc(), img[0] - 10, p[1])
    # projection left of the image
    X, p = settle(back_project(-0.5, 700, 3.0, *poses[0]), poses)
    add_from(X, rand_desc(), "x_negative")
    add_to(rand_desc(), 3.0, p[1])
    # behind the camera: projects into the image through the negative depth
    X, p = settle(back_project(760, 800, -3.0, *poses[0]), poses)
    assert 0 <= p[0] < img[0] - 1 and 0 <= p[1] < img[1] - 1
    add_from(X, rand_desc(), "behind")
    add_to(rand_desc(), p[0] + 3, p[1])
    # NaN point, with an exact copy of its descriptor among the keypoints
    dn = rand_desc()
    add_from(np.full(3, np.nan, np.float32), dn, "nan")
    add_to(dn, 760, 900)

    n_edge = len(from_d)
    twins = [d for d, name in zip(from_d, list(expect)) if name != "nan"]
    D = np.concatenate([d0] + from_d + twins)
    XX = np.concatenate([x0, np.stack(from_x), np.full((len(twins), 3), np.nan, np.float32)])
    DT = np.concatenate([dt0] + to_d)
    UV = np.concatenate([uv0, np.stack(to_uv)])
    assert len(D) == 300 + n_edge + len(twins)

    # the added rows leave the global matching, and so the first pass, as it was
    o1b = orc.verify_pair_cov(D, XX, DT, UV, K4, image_size=img)
    assert np.array_equal(o1b["matches"], o1["matches"]) and o1b["rvec"].tobytes() == o1["rvec"].tobytes()
    cap = len(D)
    g1b = batch(eng, [(D, XX)], [(DT, UV)], cap, dim, repeat_once=False, img=img)[0]
    assert np.array_equal(g1b["matches"], g1["matches"]) and g1b["rvec"].tobytes() == g1["rvec"].tobytes()

    sel, _ = orc.guess_match(D, XX, DT, UV, K4, *poses[0], image_size=img, guess_win_size=WIN)
    for name, (i, j) in expect.items():
        assert sel[i] == (-1 if j is None else j), (name, sel[i], j)
    o = orc.verify_pair_repeat(D, XX, DT, UV, K4, image_size=img, guess_win_size=WIN)
    g = batch(eng, [(D, XX)], [(DT, UV)], cap, dim, img=img)[0]
    assert_oracle(g, o, dim)
    got = set(g["matches"].tolist())
    for name, (i, j) in expect.items():
        assert (i in got) == (j is not None), name
    assert second_pass_changed(D, XX, DT, UV, o, img)

    # words3B: the TO keypoints' own 3-D points (a fifth missing) drive the covariance of the second pass's correspondences
    z = rng.uniform(0.5, 5, len(UV)).astype(np.float32)
    XT = np.stack([(UV[:, 0] - K4[2]) * z / K4[0], (UV[:, 1] - K4[3]) * z / K4[1], z], 1).astype(np.float32)
    XT[::5] = np.nan
    o3 = orc.verify_pair_repeat(D, XX, DT, UV, K4, xyz_to=XT, image_size=img, guess_win_size=WIN)
    assert len(DT) <= cap
    T3 = np.zeros((1, cap, dim), np.uint8)
    U3 = np.zeros((1, cap, 2), np.float32)
    X3 = np.full((1, cap, 3), np.nan, np.float32)
    T3[0, :len(DT)], U3[0, :len(DT)], X3[0, :len(DT)] = DT, UV, XT
    g3 = eng.verify_batch(D[None], XX[None], T3, U3, K4, [cap], [len(DT)], xyz_to=X3, image_size=img, repeat_once=True, guess_win_size=WIN)[0]
    assert_oracle(g3, o3, ("words3B", dim))
    assert o3["ok"] and o3["covariance"].tobytes() != o["covariance"].tobytes()
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- size edges
def match_smem(cap, nw):
    return 64 * (8 * nw + 8) * 4 + cap * (4 + 4 + 4 + 2 + 2 + 1 + 1 + 4 + 4 + 2 + 2) + 2 * cap * nw * 4 + 128  # verify.cuh match_smem_bytes


def guess_smem(cap):
    return cap * (8 + 4 + 4 + 2 + 2 + 1) + 64  # guess_smem_bytes


def pnp_smem(cap):
    return cap * (12 + 8 + 4 + 4 + 2 + 2 + 1) + 320 * 12 + 128 * (4 + 6 * 8) + (28 * 32 + 32) * 8 + 1024  # pnp_smem_bytes


def from_dict_smem(rows, nw):
    return rows * (nw * 4 + 4 + 4 + 4 + 2 + 2 + 1 + 1) + 128  # from_dict_smem_bytes


def largest_cap(eng, dim):
    import torch

    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    nw = dim // 4
    st = [eng.verify_static_smem(k) for k in range(4)]
    assert st[0] > 0  # resolve_rounds' tables

    def fits(c):
        return (st[0] + match_smem(c, nw) <= optin and st[1] + guess_smem(c) <= optin and st[2] + pnp_smem(c) <= optin
                and st[3] + from_dict_smem(c, nw) <= optin)

    top = max(c for c in range(1, 4097) if fits(c))
    assert top < 4096 and not fits(top + 1)
    return top


@pytest.mark.parametrize("dim", DIMS)
def test_size_edges_of_the_matching_kernel(dim):
    """nf = nt on both sides of the 1024-thread CTA and at the largest cap the engine accepts, through lcd_verify_batch and the fused
    query with the second pass on; one more is LCD_ERR_CAPACITY, and the engine then runs a valid call as before."""
    rng = np.random.default_rng(90 + dim)
    eng = Engine(desc_dim=dim)
    top = largest_cap(eng, dim)
    small = None
    changed = 0
    for n in (1023, 1024, 1025, top):
        d, x, q, uv, _ = make_scene(rng, n, n, dim, flip=0.08, outlier_frac=0.3)
        o = orc.verify_pair_repeat(d, x, q, uv, K4, image_size=IMG, guess_win_size=WIN)
        g = batch(eng, [(d, x)], [(q, uv)], n, dim)[0]
        assert_oracle(g, o, n)
        assert o["ok"], n
        changed += second_pass_changed(d, x, q, uv, o)
        fe = Engine(desc_dim=dim)
        fe.sig_add_batch([7], d[None], x[None])
        r = Fused(fe, [(q, uv)]).run([7], [7], vparams())
        assert_same_bits(r[0], g, n)
        fe.close()
        if small is None:
            small = (d, x, q, uv, g)
    assert changed >= 3, changed

    c = top + 1
    z = np.zeros((1, c, dim), np.uint8)
    with pytest.raises(LcdError) as ex:
        eng.verify_batch(z, np.zeros((1, c, 3), np.float32), z, np.zeros((1, c, 2), np.float32), K4, [c], [c], image_size=IMG,
                         repeat_once=True, guess_win_size=WIN)
    assert ex.value.code == LCD_ERR_CAPACITY
    d, x, q, uv, g = small
    again = batch(eng, [(d, x)], [(q, uv)], len(d), dim)[0]
    assert np.array_equal(again["matches"], g["matches"]) and np.array_equal(again["inliers"], g["inliers"])
    assert again["rvec"].tobytes() == g["rvec"].tobytes() and again["covariance"].tobytes() == g["covariance"].tobytes()

    fe = Engine(desc_dim=dim)
    fe.sig_add_batch([7], z, np.zeros((1, c, 3), np.float32))
    with pytest.raises(LcdError) as ex:
        Fused(fe, [(z[0], np.zeros((c, 2), np.float32))]).run([7], [7], vparams())
    assert ex.value.code == LCD_ERR_CAPACITY
    again = batch(fe, [(d, x)], [(q, uv)], len(d), dim)[0]
    assert again["rvec"].tobytes() == g["rvec"].tobytes() and np.array_equal(again["matches"], g["matches"])
    fe.close()
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- lcd_process_frames
K4S = (262.5, 262.5, 160.0, 120.0)  # the 320 x 240 frames of synth.make_place_world
IMG_S = (320, 240)
N_FEATURES = 1000


@pytest.fixture(scope="module")
def orb_world():
    """five places, 120 signatures, six 320 x 240 views (keypoints as cv::ORB finds them, fewer than N_FEATURES), one of them textureless"""
    from oracle import feature2d_py as f2d

    p = f2d.OrbParams(n_features=600)
    world = synth.make_place_world(lambda img, dep: f2d.detect_describe(img, dep, K4, p), n_places=5, n_words=2800, n_signatures=120, feats=600,
                                   height=240, width=320, seed=9)
    imgs, deps, places = synth.make_view_frames(world, 6, seed=5, max_shift=4)
    imgs[3] = 7
    return world, imgs, deps


def orb_engine(world):
    eng = Engine(max_words=8192, max_signatures=400)
    eng.add_words(world.word_ids, world.vocab)
    eng.last_word_id = int(world.word_ids.max())
    eng.update()
    eng.load_csr(world.smap.word_ids, world.smap.row_ptr, world.smap.sig, world.smap.cnt)
    eng.set_ni(world.smap.sig_ids, world.smap.ni)
    eng.sig_add_batch(world.smap.sig_ids, world.store.desc, world.store.xyz, world.smap.ni)
    return eng


def test_process_frames_second_pass_with_frame_counts_and_words3B(orb_world):
    """lcd_process_frames: TO rows with per-frame keypoint counts and the frames' own 3-D points (words3B) for the covariance, against
    verify_pair_repeat(xyz_to = the ORB points) and lcd_verify_batch with the same xyz_to."""
    from oracle import feature2d_py as f2d

    world, imgs, deps = orb_world
    sig_ids = world.smap.sig_ids
    eng = orb_engine(world)
    op = Engine.orb_params(K4S, n_features=N_FEATURES)
    nkp, _, _, hyp, res = eng.process_frames(imgs, deps, op, sig_ids, len(sig_ids) + 1, vparams(True, IMG_S, K4S))
    _, _, _, hyp1, res1 = eng.process_frames(imgs, deps, op, sig_ids, len(sig_ids) + 1, vparams(False, IMG_S, K4S))
    assert np.array_equal(hyp, hyp1)
    vb = Engine()
    changed = 0
    for b in range(len(imgs)):
        kp, d, x = f2d.detect_describe(imgs[b], deps[b], K4S, f2d.OrbParams(n_features=N_FEATURES))
        assert nkp[b] == len(kp)
        if len(kp) == 0:
            assert not res[b]["ok"] and res[b]["n_matches"] == 0
            continue
        row = int(np.flatnonzero(sig_ids == hyp[b])[0])
        n = int(world.smap.ni[row])
        fd, fx = world.store.desc[row][:n], world.store.xyz[row][:n]
        o = orc.verify_pair_repeat(fd, fx, d, kp[:, :2], K4S, xyz_to=x, image_size=IMG_S, guess_win_size=WIN)
        assert_oracle(res[b], o, b)
        g = batch(vb, [(fd, fx)], [(d, kp[:, :2])], max(n, len(kp)), 32, img=IMG_S, K=K4S, xyz_to=[x])[0]
        assert_same_bits(res[b], g, b)
        if second_pass_changed(fd, fx, d, kp[:, :2], o, IMG_S, K4S):
            changed += 1
            assert res[b]["rvec"].tobytes() != res1[b]["rvec"].tobytes(), b
    assert nkp[3] == 0 and ((nkp > 0) & (nkp < N_FEATURES)).any()
    assert changed >= 2, changed
    vb.close()
    eng.close()


def test_sharded_step_second_pass_equals_the_unsharded_call(orb_world, monkeypatch):
    """lcd_shard_process_frames_dev on a communicator of one rank with Reg/RepeatOnce on: hypotheses and registrations bit for bit those
    of lcd_process_frames_dev on the same engine."""
    import torch

    world, imgs, deps = orb_world
    monkeypatch.setenv("LCD_SHARD_SCORE_PARTS", "2")
    eng = orb_engine(world)
    sm = world.smap
    op = Engine.orb_params(K4S, n_features=N_FEATURES)
    vp = vparams(True, IMG_S, K4S)
    nf, ns = len(imgs), len(sm.sig_ids)
    d_img = torch.from_numpy(imgs).cuda()
    d_dep = torch.from_numpy(deps.view(np.int16)).cuda()
    d_sig = torch.from_numpy(sm.sig_ids).cuda()
    d_rowids = torch.from_numpy(world.word_ids).cuda()
    ext = torch.cuda.ExternalStream(eng.stream)
    with torch.cuda.stream(ext):
        w0 = torch.zeros(nf * N_FEATURES, dtype=torch.int32, device="cuda")
        l0 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        eng.process_frames_dev(d_img.data_ptr(), nf, 320, 240, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, ns + 1, vp, w0.data_ptr(),
                               l0.data_ptr(), True, 0.8, True)
        hyp0, res0 = eng.process_fetch(nf)
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        w1 = torch.zeros(nf * N_FEATURES, dtype=torch.int32, device="cuda")
        l1 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        eng.shard_process_frames_dev(d_img.data_ptr(), nf, 320, 240, 3, d_dep.data_ptr(), 1, op, d_sig.data_ptr(), ns, ns + 1, d_rowids.data_ptr(),
                                     int(world.word_ids.max()), vp, w1.data_ptr(), l1.data_ptr(), True, 0.8, True)
        hyp1, res1 = eng.process_fetch(nf)
        eng.shard_comm_destroy()
    assert torch.equal(w0, w1) and torch.equal(l0, l1) and np.array_equal(hyp0, hyp1)
    assert sum(r["ok"] for r in res0) >= 4
    for b, (a, c) in enumerate(zip(res0, res1)):
        assert a["ok"] == c["ok"] and a["n_matches"] == c["n_matches"] and a["n_inliers"] == c["n_inliers"], b
        assert all(a[k].tobytes() == c[k].tobytes() for k in ("rvec", "tvec", "transform", "covariance")), b
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- decided frames, proximity
from test_gpu_proximity import F as PF, S as PS, frames as px_frames, make_engine as px_engine, scene as px_scene  # noqa: E402
from test_gpu_proximity import set_map as px_set_map, world  # noqa: E402,F401  (world: the module fixture of that file's map)


def f32_norm(T):
    x, y, z = (np.float32(v) for v in np.asarray(T, np.float32)[:, 3])
    return np.float32(np.sqrt(np.float32(np.float32(np.float32(x * x) + np.float32(y * y)) + np.float32(z * z))))


def store_row(st, h):
    """the signature-store row of place h (places past the store have no row: nothing to register)"""
    return (st.desc[h - 1], st.xyz[h - 1]) if h <= PS else (st.desc[0][:0], st.xyz[0][:0])


def oracle_reg(st, h, fq, fu, repeat, img):
    d, x = store_row(st, h)
    if repeat:
        return orc.verify_pair_repeat(d, x, fq, fu, K4, image_size=img, guess_win_size=WIN)
    o = orc.verify_pair_cov(d, x, fq, fu, K4, image_size=img)
    o["second_pass"] = False
    return o


def test_decided_frames_follow_the_second_pass(world):
    """lcd_decide_batch_dev then lcd_verify_decided_dev: the final status and loop id of every accepted frame follow from the oracle's
    registration of the pass in force — with a 128 x 96 image most projections fall outside, so pass 1 succeeds and pass 2 fails, and
    RGBD/MaxLoopClosureDistance sits between the two passes' translation norms of one frame."""
    import torch
    from oracle import decide_py as dc

    vocab, wid, m, st, q, uv, places = world
    n_places, B = 1000, 48
    ids, poses, nbr, ptr, flat = px_scene(n_places)
    eng = px_engine(world, n_places, B)
    px_set_map(eng, ids)
    _, raw, flags, _ = px_frames(world, ids, poses, B, seed=31)
    d_like = torch.from_numpy(raw.reshape(-1)).cuda()
    d_q = torch.from_numpy(np.ascontiguousarray(q[:B * PF]).reshape(-1)).cuda()
    d_uv = torch.from_numpy(np.ascontiguousarray(uv[:B * PF]).reshape(-1)).cuda()
    torch.cuda.synchronize()
    fr = lambda b: (q[b * PF:(b + 1) * PF], uv[b * PF:(b + 1) * PF])

    def decided(vp, max_dist):
        eng.clients_create(B)
        eng.decide_batch_dev(d_like.data_ptr(), B, len(ids), np.arange(B), flags, Engine.decide_params(max_loop_closure_distance=max_dist))
        d0 = eng.decide_fetch(B)
        eng.verify_decided_dev(d_q.data_ptr(), d_uv.data_ptr(), B, PF, vp)
        _, res = eng.process_fetch(B)
        return d0, res, eng.decide_fetch(B)

    d0, _, _ = decided(vparams(True), 0.0)
    acc = [b for b in range(B) if int(d0[b]["status"]) == dc.ACCEPTED and int(d0[b]["loop_id"]) <= PS]
    assert len(acc) >= 5, len(acc)
    max_dist = None
    for b in acc:
        h = int(d0[b]["loop_id"])
        o1, o2 = oracle_reg(st, h, *fr(b), False, IMG), oracle_reg(st, h, *fr(b), True, IMG)
        if o1["ok"] and o2["ok"]:
            n1, n2 = sorted((f32_norm(o1["transform"]), f32_norm(o2["transform"])))
            mid = np.float32((np.float64(n1) + np.float64(n2)) / 2)
            if n1 < mid < n2:
                max_dist = float(mid)
                break
    assert max_dist is not None

    vb = Engine()
    final, changed = {}, 0
    for img in (IMG, (128, 96)):
        for repeat in (False, True):
            d0, res, d2 = decided(vparams(repeat, img), max_dist)
            acc = [b for b in range(B) if int(d0[b]["status"]) == dc.ACCEPTED]
            g = batch(vb, [store_row(st, int(d0[b]["loop_id"])) for b in acc], [fr(b) for b in acc], PF, 32, repeat_once=repeat, img=img)
            for k, b in enumerate(acc):
                h = int(d0[b]["loop_id"])
                o = oracle_reg(st, h, *fr(b), repeat, img)
                assert_oracle(res[b], o, (img, repeat, b))
                assert_same_bits(res[b], g[k], (img, repeat, b))
                status, loop = dc.ACCEPTED, h
                if not o["ok"]:
                    status, loop = dc.VERIFY_REJECTED, 0
                elif f32_norm(o["transform"]) > np.float32(max_dist):
                    status, loop = dc.DISTANCE_REJECTED, 0
                assert (int(d2[b]["status"]), int(d2[b]["loop_id"])) == (status, loop), (img, repeat, b)
                final[(img, repeat, b)] = (status, o["ok"])
                if repeat and img == IMG:
                    changed += second_pass_changed(*store_row(st, h), *fr(b), o)
    keys = [k[2] for k in final if k[:2] == (IMG, True)]
    assert any(final[(IMG, False, b)][0] != final[(IMG, True, b)][0] for b in keys)                      # the distance test
    assert any(final[((128, 96), False, b)][1] and not final[((128, 96), True, b)][1] for b in keys)  # pass 1 ok, pass 2 fails
    assert changed >= 2, changed
    vb.close()
    eng.close()


def test_proximity_registrations_follow_the_second_pass(world):
    """lcd_decide_proximity_dev: every attempted registration (store row through px_slot, frame row through px_row) equals
    lcd_verify_batch bit for bit and the oracle's second pass; accepted links, link types, suppression and the decision follow from
    px.apply on the oracle's second-pass results."""
    import torch
    from oracle import decide_py as dc
    from oracle import proximity_py as px

    vocab, wid, m, st, q, uv, places = world
    n_places, B = 1000, 37
    ids, poses, nbr, ptr, flat = px_scene(n_places)
    eng = px_engine(world, n_places, B)
    px_set_map(eng, ids)
    eng.clients_set_map_poses(ids, poses, ptr, flat)
    fp, raw, flags, enabled = px_frames(world, ids, poses, B, seed=n_places + B)
    d_like = torch.from_numpy(raw.reshape(-1)).cuda()
    d_q = torch.from_numpy(np.ascontiguousarray(q[:B * PF]).reshape(-1)).cuda()
    d_uv = torch.from_numpy(np.ascontiguousarray(uv[:B * PF]).reshape(-1)).cuda()
    torch.cuda.synchronize()
    adj = eng.adjust_likelihood(raw)
    pose_of = {int(i): poses[k] for k, i in enumerate(ids)}
    vb = Engine()
    recs, changed, n_checked = {}, 0, 0
    for repeat in (False, True):
        eng.clients_create(B)
        eng.decide_batch_dev(d_like.data_ptr(), B, len(ids), np.arange(B), flags, Engine.decide_params())
        d0 = eng.decide_fetch(B)
        eng.decide_proximity_dev(d_q.data_ptr(), d_uv.data_ptr(), B, PF, fp, enabled, Engine.proximity_params(vparams(repeat)))
        rec, d1 = eng.proximity_fetch(B), eng.decide_fetch(B)
        recs[repeat] = rec
        for b in range(B):
            if not enabled[b]:
                continue
            use = not flags[b] & (dc.FRAME_SKIP | dc.FRAME_HOLD)
            like = {int(i): adj[b][k + 1] for k, i in enumerate(ids)} if use else {}
            nearest, paths, attempts = px.detect(fp[b], pose_of, nbr, like)
            r = rec[b]
            assert r["n_attempts"] == len(attempts), b
            fq, fu = q[b * PF:(b + 1) * PF], uv[b * PF:(b + 1) * PF]
            results = []
            for g in r["paths"]:
                h = g["candidate_id"]
                if h > PS:
                    assert not g["result"]["ok"] and g["result"]["n_matches"] == 0
                    results.append((False, g["result"]["transform"]))
                    continue
                o = oracle_reg(st, h, fq, fu, repeat, IMG)
                gb = batch(vb, [(st.desc[h - 1], st.xyz[h - 1])], [(fq, fu)], PF, 32, repeat_once=repeat)[0]
                assert_oracle(g["result"], o, (repeat, b, h))
                assert_same_bits(g["result"], gb, (repeat, b, h))
                results.append((o["ok"], o["transform"] if o["ok"] else g["result"]["transform"]))
                n_checked += 1
                if repeat:
                    changed += second_pass_changed(st.desc[h - 1], st.xyz[h - 1], fq, fu, o)
            acc, types, sup, loop, status, _ = px.apply(nearest, attempts, results, int(d0[b]["loop_id"]), int(d0[b]["status"]), 1.0, 0.0)
            assert [g["accepted"] for g in r["paths"]] == acc and [g["link_type"] for g in r["paths"]] == types, b
            assert r["suppressed_id"] == sup and (int(d1[b]["loop_id"]), int(d1[b]["status"])) == (loop, status), b
    assert n_checked >= 20 and changed >= 3, (n_checked, changed)
    differ = [b for b in range(B) if [(g["result"]["n_matches"], g["result"]["transform"].tobytes()) for g in recs[False][b]["paths"]]
              != [(g["result"]["n_matches"], g["result"]["transform"].tobytes()) for g in recs[True][b]["paths"]]]
    assert differ
    vb.close()
    eng.close()
