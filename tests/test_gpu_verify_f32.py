"""Geometric verification on float-descriptor engines (LCD_DESC_F32, 64-D and 128-D): RegistrationVis global matching through a
temporary dictionary with squared L2 in rtflann's order, PnP, and the Reg/RepeatOnce pass, through every store-backed caller.

References: the CPU oracle (verify_pair_repeat / verify_pair_cov with desc_type 1, its float matching pinned to the reference's
rtflann and cv::BFMatcher by test_oracle_verify_f32.py): correspondence and inlier word ids exact, ok and iterations exact, pose /
transform / covariance 1e-4; and lcd_verify_batch on the same pair, bit for bit, for the store-backed calls."""
import numpy as np
import pytest

from oracle import oracle_py as orc
from rtabmap_b200 import Engine, synth
from rtabmap_b200.capi import LCD_DESC_F32

pytestmark = pytest.mark.gpu

K4 = synth.CAMERA_K4
IMG = (640, 480)
WIN = 40
DIMS = [64, 128]


def unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def rand_desc(rng, n, dim):
    return unit(rng.laplace(0.0, 1.0, (n, dim)))


def near(rng, desc, r):
    """unit vectors about r away from desc (squared distance ~ r^2; unrelated unit vectors are ~2 apart)"""
    return unit(desc + (r / np.sqrt(desc.shape[1])) * rng.standard_normal(desc.shape))


def make_scene(rng, nf, nt, dim, noise=0.5, outlier_frac=0.3, nan_every=40):
    """FROM points seen from a random pose and a TO view of them.  FROM holds near-duplicate pairs (words created and matched inside
    the FROM frame, then seen twice), TO holds near-duplicates of each other (TO new words matched by later TO descriptors) and
    descriptors midway between two FROM descriptors (NNDR rejections).  Returns desc, xyz, desc_to, uv_to, xyz_to."""
    rv, tv = rng.normal(0, 0.08, 3), rng.normal(0, 0.15, 3)
    R = synth.rodrigues(rv)
    px = np.stack([rng.uniform(10, IMG[0] - 10, nf), rng.uniform(10, IMG[1] - 10, nf)], 1)
    z = rng.uniform(0.8, 6.0, nf)
    cam = np.stack([(px[:, 0] - K4[2]) * z / K4[0], (px[:, 1] - K4[3]) * z / K4[1], z], 1)
    X = ((cam - tv) @ R).astype(np.float32)
    if nan_every and nf:
        X[::nan_every] = np.nan
    desc = rand_desc(rng, nf, dim)
    k = nf // 12
    if k:
        i = rng.permutation(nf)[:2 * k]
        desc[i[:k]] = near(rng, desc[i[k:]], 0.1)
    m = min(nf, nt)
    desc_to = rand_desc(rng, nt, dim)
    uv_to = np.stack([rng.uniform(0, IMG[0], nt), rng.uniform(0, IMG[1], nt)], 1)
    if m:
        uv = orc.project_points(np.nan_to_num(X), K4, rv, tv) + rng.normal(0, 0.5, (nf, 2))
        src, at = rng.permutation(nf)[:m], rng.permutation(nt)[:m]
        desc_to[at] = near(rng, desc[src], noise)
        uv_to[at] = uv[src]
        bad = at[rng.random(m) < outlier_frac]
        uv_to[bad] = np.stack([rng.uniform(0, IMG[0], len(bad)), rng.uniform(0, IMG[1], len(bad))], 1)
        mid = at[rng.random(m) < 0.05]
        if nf >= 2:
            a, b = rng.integers(0, nf, (2, len(mid)))
            desc_to[mid] = unit(desc[a] + desc[b])
    kt = nt // 15
    if kt:
        j = rng.permutation(nt)[:2 * kt]
        desc_to[j[:kt]] = near(rng, desc_to[j[kt:]], 0.1)
    xyz_to = (rng.uniform(-2, 2, (nt, 3)) + [0, 0, 4]).astype(np.float32)
    xyz_to[::7] = np.nan
    return desc, X, desc_to, uv_to.astype(np.float32), xyz_to


def float_engine(dim):
    return Engine(desc_type=LCD_DESC_F32, desc_dim=dim)


def batch(eng, rows, frames, cap, dim, repeat_once=True, xyz_to=None, nndr=0.8):
    """lcd_verify_batch of FROM rows[b] = (desc, xyz) against frames[b] = (desc, uv), staged at stride cap"""
    B = len(rows)
    F = np.zeros((B, cap, dim), np.float32)
    T = np.zeros((B, cap, dim), np.float32)
    X = np.full((B, cap, 3), np.nan, np.float32)
    U = np.zeros((B, cap, 2), np.float32)
    XT = None if xyz_to is None else np.full((B, cap, 3), np.nan, np.float32)
    for b, ((d, x), (q, uv)) in enumerate(zip(rows, frames)):
        F[b, :len(d)], X[b, :len(d)] = d, x
        T[b, :len(q)], U[b, :len(q)] = q, uv
        if xyz_to is not None:
            XT[b, :len(q)] = xyz_to[b]
    return eng.verify_batch(F, X, T, U, K4, [len(d) for d, _ in rows], [len(q) for q, _ in frames], image_size=IMG, xyz_to=XT,
                            repeat_once=repeat_once, guess_win_size=WIN, nndr=nndr)


def oracle(d, x, q, uv, repeat_once=True, xyz_to=None, nndr=0.8):
    return orc.verify_pair_repeat(d, x, q, uv, K4, xyz_to=xyz_to, nndr=nndr, image_size=IMG, repeat_once=repeat_once, guess_win_size=WIN)


def first_pass_iterations(d, x, q, uv, nndr=0.8):
    """RANSAC iterations of the global-matching pass, from the oracle's correspondences (None: PnP is not run)"""
    fid, tid = orc.match_pair(d, q, nndr)
    o = orc.verify_pair_cov(d, x, q, uv, K4, nndr=nndr, image_size=IMG)
    if len(o["matches"]) < 20:
        return None
    fi = [int(np.flatnonzero(fid == w)[0]) for w in o["matches"]]
    ti = [int(np.flatnonzero(tid == w)[0]) for w in o["matches"]]
    return orc.pnp_ransac(x[fi], uv[ti], K4, guess=np.zeros(6))[4]


def second_pass_changed(d, x, q, uv, o):
    """True when the oracle's second pass ran and chose another set of FROM points than its global matching did."""
    if not o["second_pass"]:
        return False
    o1 = orc.verify_pair_cov(d, x, q, uv, K4, image_size=IMG)
    fid, _ = orc.match_pair(d, d[:0])
    return sorted(int(np.flatnonzero(fid == w)[0]) for w in o1["matches"]) != o["matches"].tolist()


def matching_branches(d, q, nndr=0.8):
    """Which branches of the temporary dictionary the oracle's matching of (d, q) takes: FROM descriptors matched to a word created
    earlier in the FROM frame, TO descriptors rejected by the NNDR test (new words: with two or more FROM words every TO descriptor has
    two index hits), and TO descriptors matched to a word created earlier in the TO frame."""
    fid, tid = orc.match_pair(d, q, nndr)
    n_words = int(fid.max()) if len(fid) else 0
    new_t = tid[tid > n_words]
    return {"from_dependency": len(np.unique(fid)) < len(fid), "to_nndr_rejection": n_words >= 2 and len(new_t) > 0,
            "to_dependency": len(np.unique(new_t)) < len(new_t)}


def assert_oracle(g, o, tag):
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
    """r: a result of a store-backed call, g: lcd_verify_batch's result for the same pair"""
    n_m = r["n_matches"] if "n_matches" in r else len(r["matches"])
    n_i = r["n_inliers"] if "n_inliers" in r else len(r["inliers"])
    assert r["ok"] == g["ok"] and n_m == len(g["matches"]) and n_i == len(g["inliers"]), tag
    assert r["iterations_run"] == g["iterations_run"], tag
    for k in ("rvec", "tvec", "transform", "covariance"):
        assert r[k].tobytes() == g[k].tobytes(), (tag, k)


# ---------------------------------------------------------------------------------------------------------------- lcd_verify_batch
@pytest.mark.parametrize("dim", DIMS)
def test_verify_batch_matches_oracle(dim):
    """Uneven per-pair counts (including empty sides) and NaN depths in one batch; the second pass on and off, words3B given or not."""
    rng = np.random.default_rng(dim)
    counts = [(300, 300), (250, 420), (420, 180), (150, 500), (60, 60), (0, 50), (50, 0), (500, 500)]
    scenes = [make_scene(rng, nf, nt, dim, noise=0.5 + 0.1 * (i % 3)) for i, (nf, nt) in enumerate(counts)]
    rows = [(s[0], s[1]) for s in scenes]
    frames = [(s[2], s[3]) for s in scenes]
    for branch in ("from_dependency", "to_nndr_rejection", "to_dependency"):
        assert sum(matching_branches(s[0], s[2])[branch] for s in scenes) >= 4, branch
    eng = float_engine(dim)
    changed = 0
    for repeat in (False, True):
        for with_xyz_to in (False, True):
            xt = [s[4] for s in scenes] if with_xyz_to else None
            g = batch(eng, rows, frames, 500, dim, repeat_once=repeat, xyz_to=xt)
            for b, s in enumerate(scenes):
                o = oracle(s[0], s[1], s[2], s[3], repeat, s[4] if with_xyz_to else None)
                assert_oracle(g[b], o, (repeat, with_xyz_to, b))
                if not repeat:
                    it = first_pass_iterations(s[0], s[1], s[2], s[3])
                    assert g[b]["iterations_run"] == (it if it is not None else 0), (b, g[b]["iterations_run"], it)
                elif not with_xyz_to:
                    changed += second_pass_changed(s[0], s[1], s[2], s[3], o)
    assert sum(r["ok"] for r in g) >= 4
    assert changed >= 1, changed
    eng.close()


@pytest.mark.parametrize("dim", DIMS)
def test_ties_and_duplicates_match_oracle(dim):
    """Identical descriptors inside FROM, inside TO and across the two sides: equal distances everywhere, resolved to the lowest word."""
    rng = np.random.default_rng(100 + dim)
    d, x, q, uv, _ = make_scene(rng, 300, 300, dim)
    d[10:14] = d[3]            # four exact copies inside FROM
    q[0:40] = d[100:140]       # exact copies across the sides (distance 0)
    q[50:56] = q[49]           # exact copies inside TO
    q[60] = d[7]
    q[61] = d[7]               # two TO copies of one FROM descriptor
    q[70] = unit((d[20] + d[21])[None])[0]   # equidistant from two FROM words
    eng = float_engine(dim)
    for nndr in (0.8, 0.6):
        g = batch(eng, [(d, x)] * 2, [(q, uv), (q[::-1].copy(), uv[::-1].copy())], 300, dim, nndr=nndr)
        for b, (qq, uu) in enumerate([(q, uv), (q[::-1].copy(), uv[::-1].copy())]):
            assert_oracle(g[b], oracle(d, x, qq, uu, nndr=nndr), (nndr, b))
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- size edges
@pytest.mark.parametrize("dim", DIMS)
def test_size_edges_up_to_4096(dim):
    """Counts 0, 1, 31, 32, 33, 1000 and 4096 per side with cap 4096: no capacity refusal, every pair equals the oracle."""
    rng = np.random.default_rng(200 + dim)
    eng = float_engine(dim)
    for which in range(4):
        assert eng.verify_static_smem(which) >= 0
    counts = [(0, 0), (1, 1), (31, 33), (32, 32), (33, 31), (1000, 1000), (4096, 4096), (0, 4096)]
    scenes = [make_scene(rng, nf, nt, dim) for nf, nt in counts]
    g = batch(eng, [(s[0], s[1]) for s in scenes], [(s[2], s[3]) for s in scenes], 4096, dim)
    for b, s in enumerate(scenes):
        assert_oracle(g[b], oracle(*s[:4]), counts[b])
    assert g[5]["ok"] and g[6]["ok"]
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- signature store
class Fused:
    """lcd_verify_top_dev with one-hot likelihood rows: frame b is registered against signature pick[b] of the store."""

    def __init__(self, eng, frames):
        import torch

        self.torch, self.eng, self.B, self.nq = torch, eng, len(frames), len(frames[0][0])
        q = np.concatenate([f[0] for f in frames])
        uv = np.concatenate([f[1] for f in frames]).astype(np.float32)
        self.d_q = torch.from_numpy(np.ascontiguousarray(q).reshape(-1)).cuda()
        self.d_uv = torch.from_numpy(uv.reshape(-1)).cuda()

    def run(self, sig_ids, pick, nndr=0.8):
        torch = self.torch
        like = np.zeros((self.B, len(sig_ids)), np.float32)
        col = {int(s): k for k, s in enumerate(sig_ids)}
        for b, h in enumerate(pick):
            like[b, col[int(h)]] = 1.0
        d_l = torch.from_numpy(like.reshape(-1)).cuda()
        d_s = torch.from_numpy(np.asarray(sig_ids, np.int32)).cuda()
        torch.cuda.synchronize()
        vp = Engine.verify_params(K4, nndr=nndr, image_size=IMG, repeat_once=True, guess_win_size=WIN)
        self.eng.verify_top_dev(self.d_q.data_ptr(), self.d_uv.data_ptr(), self.B, self.nq, d_l.data_ptr(), d_s.data_ptr(), len(sig_ids), vp)
        hyp, res = self.eng.process_fetch(self.B)
        assert list(hyp) == [int(h) for h in pick]
        return res


@pytest.mark.parametrize("dim", DIMS)
def test_fused_query_equals_verify_batch_through_the_store_life_cycle(dim):
    """lcd_sig_add_batch with float rows, then lcd_verify_top_dev: equal to lcd_verify_batch bit for bit, on the first call (dictionary
    built) and the second (cached); a rewritten row, a freed and reused slot and a new NNDR each rebuild the dictionary."""
    rng = np.random.default_rng(300 + dim)
    st_cap, nq = 300, 360
    sc = [make_scene(rng, st_cap, nq, dim, noise=0.5 + 0.1 * i) for i in range(4)]
    store = {s + 1: (sc[s][0], sc[s][1]) for s in range(4)}
    n_row = {1: st_cap, 2: st_cap - 37, 3: st_cap, 4: st_cap}
    frames = [(sc[0][2], sc[0][3]), (sc[1][2], sc[1][3]), (sc[2][2], sc[2][3]), (sc[3][2], sc[3][3]), (sc[0][2], sc[0][3])]
    pick = [1, 2, 3, 4, 1]
    eng = float_engine(dim)
    vb = float_engine(dim)
    ids = [1, 2, 3, 4]
    eng.sig_add_batch(ids, np.stack([store[s][0] for s in ids]), np.stack([store[s][1] for s in ids]), [n_row[s] for s in ids])
    fused = Fused(eng, frames)

    def check(res, nndr=0.8):
        rows = [(store[h][0][:n_row[h]], store[h][1][:n_row[h]]) for h in pick]
        g = batch(vb, rows, frames, max(st_cap, nq), dim, nndr=nndr)
        for b, ((d, x), (q, uv)) in enumerate(zip(rows, frames)):
            assert_same_bits(res[b], g[b], (nndr, b))
            assert_oracle(res[b], oracle(d, x, q, uv, nndr=nndr), (nndr, b))
        return g

    r0 = fused.run(ids, pick)
    check(r0)
    r1 = fused.run(ids, pick)  # cached dictionaries
    for a, b in zip(r0, r1):
        assert_same_bits(a, {**b, "matches": np.zeros(b["n_matches"]), "inliers": np.zeros(b["n_inliers"])}, "cache")
    assert sum(r["ok"] for r in r0) >= 3

    # a row rewritten in place with another scene's descriptors
    store[1] = (sc[3][0], sc[3][1])
    eng.sig_add_batch([1], sc[3][0][None], sc[3][1][None])
    check(fused.run(ids, pick))
    # removed, then its slot reused under a new id
    eng.sig_remove(3)
    ids = [1, 2, 4, 9]
    store[9], n_row[9] = (sc[2][0][::-1].copy(), sc[2][1][::-1].copy()), st_cap
    eng.sig_add_batch([9], store[9][0][None], store[9][1][None])
    assert eng.sig_slots() == 4
    pick = [1, 2, 9, 4, 1]
    check(fused.run(ids, pick))
    # another NNDR, then back
    check(fused.run(ids, pick, 0.6), 0.6)
    check(fused.run(ids, pick, 0.8), 0.8)
    eng.close()
    vb.close()


# ---------------------------------------------------------------------------------------------------------------- process_batch
@pytest.mark.parametrize("dim", DIMS)
def test_process_batch_equals_localize_then_verify(dim):
    """lcd_process_batch and lcd_process_batch_dev on a float dictionary: word ids and likelihood equal lcd_localize_batch, the
    hypothesis is the likelihood's arg-max and its registration equals lcd_verify_batch on that pair."""
    import torch

    n_words, S, F, B = 3000, 10, 300, 6
    vocab = synth.make_float_vocabulary(n_words, dim, 5)
    ids = np.arange(1, n_words + 1, dtype=np.int32)
    m = synth.make_map(ids, S, F, seed=2)
    rng = np.random.default_rng(400 + dim)
    st_desc = near(rng, vocab[m.sig_words.reshape(-1) - 1], 0.2).reshape(S, F, dim)
    xyz = np.empty((S, F, 3), np.float32)
    z = rng.uniform(0.5, 5.0, (S, F)).astype(np.float32)
    xyz[..., 0] = rng.uniform(-0.55, 0.55, (S, F)).astype(np.float32) * z
    xyz[..., 1] = rng.uniform(-0.40, 0.40, (S, F)).astype(np.float32) * z
    xyz[..., 2] = z
    xyz[rng.random((S, F)) < 0.02] = np.nan
    places = rng.integers(0, S, B)
    q = np.empty((B, F, dim), np.float32)
    uv = np.empty((B, F, 2), np.float32)
    for b, p in enumerate(places):
        perm = rng.permutation(F)
        q[b] = near(rng, st_desc[p][perm], 0.4)
        X = np.nan_to_num(xyz[p][perm].astype(np.float64), nan=1.0)
        rv, tv = rng.normal(0, 0.06, 3), rng.normal(0, 0.1, 3)
        uv[b] = orc.project_points(X, K4, rv, tv) + rng.normal(0, 0.5, (F, 2))
        out = rng.permutation(F)[:F // 5]
        q[b, out] = rand_desc(rng, len(out), dim)
        uv[b, out] = np.stack([rng.uniform(0, 640, len(out)), rng.uniform(0, 480, len(out))], 1)

    eng = float_engine(dim)
    eng.add_words(ids, vocab)
    eng.last_word_id = n_words
    eng.update()
    eng.load_csr(m.word_ids, m.row_ptr, m.sig, m.cnt)
    eng.sig_add_batch(m.sig_ids, st_desc, xyz)
    vp = Engine.verify_params(K4, image_size=IMG, repeat_once=True, guess_win_size=WIN)
    qf, uvf = q.reshape(B * F, dim), uv.reshape(B * F, 2)
    w_ref, l_ref = eng.localize_batch(qf, B, m.sig_ids, S + 1, incremental=False)
    words, like, hyp, res = eng.process_batch(qf, uvf, B, m.sig_ids, S + 1, vp, incremental=False)
    assert np.array_equal(words, w_ref) and np.array_equal(like.view(np.uint32), l_ref.view(np.uint32))
    assert list(hyp) == [int(m.sig_ids[np.argmax(l_ref[b])]) for b in range(B)]
    assert list(hyp) == [int(m.sig_ids[p]) for p in places]
    g = batch(eng, [(st_desc[h - 1], xyz[h - 1]) for h in hyp], [(q[b], uv[b]) for b in range(B)], F, dim)
    for b in range(B):
        assert_same_bits(res[b], g[b], b)
    assert sum(r["ok"] for r in res) >= B - 1

    d_q = torch.from_numpy(qf.reshape(-1)).cuda()
    d_uv = torch.from_numpy(uvf.reshape(-1)).cuda()
    d_s = torch.from_numpy(m.sig_ids).cuda()
    d_w = torch.zeros(B * F, dtype=torch.int32, device="cuda")
    d_l = torch.zeros(B * S, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    eng.process_batch_dev(d_q.data_ptr(), d_uv.data_ptr(), B, F, d_s.data_ptr(), S, S + 1, vp, d_w.data_ptr(), d_l.data_ptr(), incremental=False)
    hyp2, res2 = eng.process_fetch(B)
    assert np.array_equal(d_w.cpu().numpy().reshape(B, F), w_ref) and np.array_equal(d_l.cpu().numpy().reshape(B, S), l_ref)
    assert np.array_equal(hyp2, hyp)
    for b in range(B):
        assert_same_bits(res2[b], g[b], ("dev", b))
    eng.close()


# ---------------------------------------------------------------------------------------------------------------- determinism
@pytest.mark.parametrize("dim", DIMS)
def test_same_bits_at_any_batch_position_and_call(dim):
    rng = np.random.default_rng(500 + dim)
    scenes = [make_scene(rng, 400, 400, dim) for _ in range(3)]
    eng = float_engine(dim)
    rows = [(s[0], s[1]) for s in scenes]
    frames = [(s[2], s[3]) for s in scenes]
    g = batch(eng, rows, frames, 400, dim)
    for order in ([2, 0, 1], [1, 1, 2, 0, 0]):
        h = batch(eng, [rows[i] for i in order], [frames[i] for i in order], 400, dim)
        for k, i in enumerate(order):
            assert np.array_equal(h[k]["matches"], g[i]["matches"]) and np.array_equal(h[k]["inliers"], g[i]["inliers"])
            assert_same_bits(h[k], g[i], (order, k))
    eng.close()
