"""The similarity likelihood (Kp/TfIdfLikelihoodUsed=false) over word-range shards, through the C ABI.

1. Emulated shards on ONE GPU (all-gather = concatenation, all-reduce = sum), G = 2, 3, 4, binary and float engines, incremental and
   fixed dictionaries: lcd_shard_similarity_ids_dev on every shard, the per-rank pair counts and valid(s) summed here, then
   lcd_shard_similarity_finalize_dev on every rank for its own frames.  Word ids and likelihood equal one unsharded engine's
   lcd_localize_similarity_batch bit for bit.  The workload plants places whose words all sit on the first shard next to places spread
   over every shard, a listed place without postings, an id the engines do not know, the virtual place (given a descriptor row, which
   must not matter), duplicate words inside places and frames, a frame of unrelated descriptors (all new words in the incremental mode),
   a short frame with padding rows, and places with and without a global descriptor, scored once with and once without the frames'.
2. lcd_shard_localize_similarity_batch_dev on a communicator of one rank equals lcd_localize_similarity_batch_dev on the same engine,
   with and without global descriptors, with the score stage in one part and in two.
3. lcd_decide_batch_dev fed the sharded rows decides as when it is fed the unsharded rows.
4. The refusals of the new calls."""
import numpy as np
import pytest

from rtabmap_b200 import Engine, LcdError, sharding, synth
from test_gpu_proximity import set_map as decide_set_map

pytestmark = pytest.mark.gpu

LCD_DESC_F32 = 1
LCD_ERR_INVALID, LCD_ERR_CAPACITY, LCD_ERR_STATE = -1, -3, -4
W, S, F, B = 6000, 120, 100, 7
PLACE_WORDS = 80
LOCAL_PLACES = 10          # places 1..10 take their words from the first quarter of the rows: one shard for every G <= 4
EMPTY_PLACE = 6            # listed, no postings
SHORT, SHORT_N = 1, 60     # frame 1 holds 60 descriptors and 40 zero padding rows
ALL_NEW = 3                # frame 3: unrelated descriptors
GD_DIM = 40


def _desc_dim(kind):
    return 32 if kind == "binary" else 64


def _world(kind):
    rng = np.random.default_rng(11)
    vocab = synth.make_binary_vocabulary(W, 32, 21) if kind == "binary" else synth.make_float_vocabulary(W, 64, 21)
    ids = np.arange(1, W + 1, dtype=np.int32) * 2
    sig_ids = np.arange(1, S + 1, dtype=np.int32)
    place_rows = []
    for p in range(S):
        rows = rng.integers(0, W // 4 if p < LOCAL_PLACES else W, PLACE_WORDS)
        rows[:8] = rows[8:16]   # duplicate words: counts > 1 in the postings
        place_rows.append(rows)
    key = np.concatenate([ids[r].astype(np.int64) * (S + 1) + s for s, r in zip(sig_ids, place_rows) if s != EMPTY_PLACE])
    uk, cnt = np.unique(key, return_counts=True)
    w, sg = uk // (S + 1), uk % (S + 1)
    word_ids = np.unique(w).astype(np.int32)
    row_ptr = np.searchsorted(w, word_ids).astype(np.int64)
    row_ptr = np.append(row_ptr, len(w))
    csr = (word_ids, row_ptr, sg.astype(np.int32), cnt.astype(np.int32))

    q = np.empty((B, F, vocab.shape[1]), vocab.dtype)
    for f in range(B):
        rows = np.concatenate([place_rows[(f * 17) % S], rng.integers(0, W, F - PLACE_WORDS)])[rng.permutation(F)]
        d = vocab[rows]
        d = synth.flip_bits(d, 0.02, rng) if kind == "binary" else d + rng.normal(0, 0.02, d.shape).astype(np.float32)
        d[F - 6:] = d[:6]       # duplicate descriptors: the same word twice in the frame
        q[f] = d
    if kind == "binary":
        q[ALL_NEW] = rng.integers(0, 256, (F, 32), dtype=np.uint8)
    else:
        q[ALL_NEW] = synth.make_float_vocabulary(F, 64, 999)
    q[SHORT, SHORT_N:] = 0
    n_valid = np.full(B, F, np.int32)
    n_valid[SHORT] = SHORT_N

    # global descriptors (>= 0, as the reference asserts): two places in three carry one, stored in a caller table in shuffled order
    # with spare rows; the list is the virtual place, every place, and an id no engine knows
    lst = np.concatenate([[0], sig_ids, [9999]]).astype(np.int32)
    with_gd = sig_ids[sig_ids % 3 != 0]
    gd_place = np.abs(rng.normal(size=(len(with_gd), GD_DIM))).astype(np.float32)
    gd_place /= np.linalg.norm(gd_place, axis=1, keepdims=True)
    n_rows = len(with_gd) + 5
    order = rng.permutation(n_rows)
    table = np.abs(rng.normal(size=(n_rows, GD_DIM))).astype(np.float32)
    table[order[:len(with_gd)]] = gd_place
    row_of = {int(s): int(order[i]) for i, s in enumerate(with_gd)}
    row_of_k = np.array([row_of.get(int(s), -1) for s in lst], np.int32)
    row_of_k[0] = int(order[0])   # the virtual place is 0 whatever row it is given
    gd_frames = np.abs(rng.normal(size=(B, GD_DIM))).astype(np.float32)
    gd_frames /= np.linalg.norm(gd_frames, axis=1, keepdims=True)
    return dict(vocab=vocab, ids=ids, csr=csr, q=np.ascontiguousarray(q), n_valid=n_valid, lst=lst, with_gd=with_gd, gd_place=gd_place,
                table=table, row_of_k=row_of_k, gd_frames=gd_frames)


def _engine(kind, w, ids, vocab, r0=0):
    e = Engine(desc_type=LCD_DESC_F32 if kind == "float" else 0, desc_dim=_desc_dim(kind))
    e.add_words(ids, vocab)
    e.last_word_id = int(w["ids"].max())
    e.update()
    if r0:
        e.shard_set_row_offset(r0)
    e.load_csr(*sharding.shard_csr(*w["csr"], ids))
    return e


def _unsharded(kind, w):
    e = _engine(kind, w, w["ids"], w["vocab"])
    e.gdesc_add(w["with_gd"], w["gd_place"])
    return e


def _at(t, elems):
    """device address of element `elems` of a contiguous tensor"""
    return t.data_ptr() + elems * t.element_size()


@pytest.mark.parametrize("incremental", [True, False])
@pytest.mark.parametrize("kind", ["binary", "float"])
@pytest.mark.parametrize("G", [2, 3, 4])
def test_emulated_shards_equal_one_engine(G, kind, incremental):
    import torch

    w = _world(kind)
    q, n_valid, lst = w["q"], w["n_valid"], w["lst"]
    ns, last = len(lst), int(w["ids"].max())
    full = _unsharded(kind, w)
    want = {}
    for gd in (False, True):
        for b in range(B):   # per-frame calls: the reference for the short frame is the frame with only its valid descriptors
            want[gd, b] = full.localize_similarity_batch(q[b, :n_valid[b]], 1, lst, gdesc=w["gd_frames"][b:b + 1] if gd else None,
                                                         incremental=incremental)

    shards = []
    for r in range(G):
        r0, r1 = sharding.shard_rows(W, G, r)
        shards.append(_engine(kind, w, w["ids"][r0:r1], w["vocab"][r0:r1], r0))
    nq = B * F
    kw = 2 if kind == "float" else 1   # 64-bit keys on float engines
    d_q = torch.from_numpy(q.reshape(-1)).cuda()
    d_rowids = torch.from_numpy(w["ids"]).cuda()
    d_lst = torch.from_numpy(lst).cuda()
    d_nv = torch.from_numpy(n_valid).cuda()
    d_tab = torch.from_numpy(w["table"]).cuda()
    d_row = torch.from_numpy(w["row_of_k"]).cuda()
    d_fg = torch.from_numpy(w["gd_frames"]).cuda()
    torch.cuda.synchronize()
    keys = []
    for e in shards:
        k = torch.zeros(nq * 2 * kw, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        e.shard_knn2_keys_dev(d_q.data_ptr(), nq, k.data_ptr())
        e.synchronize()
        keys.append(k)
    keys_all = torch.cat(keys)          # "all-gather"
    parts = []
    for r, e in enumerate(shards):
        f0, f1 = sharding.shard_rows(B, G, r)
        w_ = torch.zeros((f1 - f0) * F, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        e.shard_resolve_frames_dev(d_q.data_ptr(), f0, f1 - f0, B, F, keys_all.data_ptr(), G, d_rowids.data_ptr(), last, d_nv.data_ptr(),
                                   w_.data_ptr(), incremental)
        e.synchronize()
        parts.append(w_)
    words_all = torch.cat(parts)        # "all-gather" of the word ids
    pairs, valid = [], []
    for e in shards:
        p = torch.full((B * ns,), -5, dtype=torch.int32, device="cuda")
        v = torch.full((ns,), -5, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        e.shard_similarity_ids_dev(words_all.data_ptr(), B, F, d_lst.data_ptr(), ns, p.data_ptr(), v.data_ptr())
        e.synchronize()
        pairs.append(p)
        valid.append(v)
    pairs_sum = torch.stack(pairs).sum(0).to(torch.int32).contiguous()   # "all-reduce(sum)"
    valid_sum = torch.stack(valid).sum(0).to(torch.int32).contiguous()
    if G >= 2:
        local = [int((p.view(B, ns)[:, 1:1 + LOCAL_PLACES] > 0).sum()) for p in pairs]
        assert local[0] > 0 and not any(local[1:]), "the places of the first quarter of the rows pair on the first shard only"
        assert all(int((v[1 + LOCAL_PLACES:1 + S] > 0).sum()) > 0 for v in valid), "spread places have postings on every shard"
    assert int(valid_sum[EMPTY_PLACE]) == 0 and int(valid_sum[0]) == 0 and int(valid_sum[-1]) == 0

    got_w = words_all.cpu().numpy().reshape(B, F)
    for gd in (False, True):
        like = torch.full((B * ns,), -1.0, dtype=torch.float32, device="cuda")
        for r, e in enumerate(shards):
            f0, f1 = sharding.shard_rows(B, G, r)
            torch.cuda.synchronize()
            e.shard_similarity_finalize_dev(_at(pairs_sum, f0 * ns), valid_sum.data_ptr(), _at(words_all, f0 * F), f1 - f0, F, d_lst.data_ptr(), ns,
                                            _at(like, f0 * ns), _at(d_fg, f0 * GD_DIM) if gd else 0, d_tab.data_ptr(), d_row.data_ptr(),
                                            len(w["table"]), GD_DIM)
            e.synchronize()
        got_l = like.cpu().numpy().reshape(B, ns)
        for b in range(B):
            want_w, want_l = want[gd, b]
            assert np.array_equal(got_w[b, :n_valid[b]], want_w[0]), f"frame {b}"
            assert not got_w[b, n_valid[b]:].any()
            assert np.array_equal(got_l[b].view(np.uint32), want_l[0].view(np.uint32)), f"frame {b}, global descriptors {gd}"
        assert not got_l[:, 0].any() and not got_l[:, -1].any()
        assert not got_l[:, EMPTY_PLACE].any() or gd and EMPTY_PLACE % 3 != 0
        if gd:
            assert (got_l[:, 1:1 + S][:, w["with_gd"] - 1] > 0.5).all()   # descriptor values (dot >= 0) where both sides carry one
        else:
            assert (got_l[np.arange(B) != ALL_NEW] > 0).any()
    if incremental:
        assert (got_w[ALL_NEW] > last).all(), "the unrelated frame is all new words"
        assert not want[False, ALL_NEW][1].any(), "new words pair with no place"


def _fused_setup(kind):
    import torch

    w = _world(kind)
    eng = _unsharded(kind, w)
    full = [b for b in range(B) if b != SHORT][:5]
    q = np.ascontiguousarray(w["q"][full])
    return w, eng, q, torch.from_numpy(np.ascontiguousarray(w["gd_frames"][full])).cuda()


@pytest.mark.parametrize("kind", ["binary", "float"])
def test_fused_similarity_with_a_single_rank_communicator_equals_the_unsharded_call(kind, monkeypatch):
    """lcd_shard_localize_similarity_batch_dev on a communicator of ONE rank: the exchanges degenerate to copies, the pipeline and its
    bookkeeping still run, and the result equals lcd_localize_similarity_batch_dev on the same engine."""
    import torch

    w, eng, q, d_fg = _fused_setup(kind)
    nf, lst = q.shape[0], w["lst"]
    ns, last = len(lst), int(w["ids"].max())
    ext = torch.cuda.ExternalStream(eng.stream)
    with torch.cuda.stream(ext):
        d_q = torch.from_numpy(q.reshape(-1)).cuda()
        d_lst = torch.from_numpy(lst).cuda()
        d_rowids = torch.from_numpy(w["ids"]).cuda()
        d_tab = torch.from_numpy(w["table"]).cuda()
        d_row = torch.from_numpy(w["row_of_k"]).cuda()
        gd_args = dict(d_frame_gdesc=d_fg.data_ptr(), d_map_gdesc=d_tab.data_ptr(), d_map_gdesc_row=d_row.data_ptr(), n_map_rows=len(w["table"]),
                       dim=GD_DIM)
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        try:
            for gd in (False, True):
                w0 = torch.zeros(nf * F, dtype=torch.int32, device="cuda")
                l0 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
                eng.localize_similarity_batch_dev(d_q.data_ptr(), nf, F, d_lst.data_ptr(), ns, d_fg.data_ptr() if gd else 0, w0.data_ptr(), l0.data_ptr())
                for parts in ("", "1", "2"):
                    if parts:
                        monkeypatch.setenv("LCD_SHARD_SCORE_PARTS", parts)
                    else:
                        monkeypatch.delenv("LCD_SHARD_SCORE_PARTS", raising=False)
                    w1 = torch.full((nf * F,), -7, dtype=torch.int32, device="cuda")
                    l1 = torch.full((nf * ns,), -1.0, dtype=torch.float32, device="cuda")
                    for _ in range(2):  # twice: the exchange buffers and events are reused
                        eng.shard_localize_similarity_batch_dev(d_q.data_ptr(), nf, F, d_lst.data_ptr(), ns, d_rowids.data_ptr(), last, w1.data_ptr(),
                                                                l1.data_ptr(), **(gd_args if gd else {}))
                    eng.synchronize()
                    assert torch.equal(w0, w1), f"word ids, LCD_SHARD_SCORE_PARTS={parts!r}, global descriptors {gd}"
                    assert torch.equal(l0.view(torch.int32), l1.view(torch.int32)), f"likelihood, LCD_SHARD_SCORE_PARTS={parts!r}, global descriptors {gd}"
                assert (l0.cpu().numpy() > 0).any()
        finally:
            eng.shard_comm_destroy()
    assert (w0.cpu().numpy() > last).any()


def test_decisions_from_the_sharded_rows_equal_the_unsharded_ones():
    """lcd_decide_batch_dev over a batch of clients: the clients fed the fused sharded step's rows reach the same decisions and posteriors
    as the clients fed lcd_localize_similarity_batch_dev's, over two steps."""
    import torch

    w, eng, q, d_fg = _fused_setup("binary")
    nf = q.shape[0]
    places = np.arange(1, S + 1, dtype=np.int32)   # the map's real places, ascending: the rows lcd_decide_batch_dev takes
    ns, last = S, int(w["ids"].max())
    eng.clients_create(2 * nf)
    decide_set_map(eng, places)
    dp = Engine.decide_params(loop_thr=0.11)
    row = w["row_of_k"][1:1 + S].copy()
    ext = torch.cuda.ExternalStream(eng.stream)
    with torch.cuda.stream(ext):
        d_q = torch.from_numpy(q.reshape(-1)).cuda()
        d_s = torch.from_numpy(places).cuda()
        d_rowids = torch.from_numpy(w["ids"]).cuda()
        d_tab = torch.from_numpy(w["table"]).cuda()
        d_row = torch.from_numpy(row).cuda()
        l0 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        l1 = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        p0 = torch.zeros(nf * (ns + 1), dtype=torch.float32, device="cuda")
        p1 = torch.zeros(nf * (ns + 1), dtype=torch.float32, device="cuda")
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        try:
            for step in range(2):
                gd = step == 1
                eng.localize_similarity_batch_dev(d_q.data_ptr(), nf, F, d_s.data_ptr(), ns, d_fg.data_ptr() if gd else 0, 0, l0.data_ptr())
                eng.shard_localize_similarity_batch_dev(d_q.data_ptr(), nf, F, d_s.data_ptr(), ns, d_rowids.data_ptr(), last, 0, l1.data_ptr(),
                                                        d_fg.data_ptr() if gd else 0, d_tab.data_ptr(), d_row.data_ptr(), len(w["table"]), GD_DIM)
                flags = np.zeros(nf, np.int32)
                eng.decide_batch_dev(l0.data_ptr(), nf, ns, np.arange(nf), flags, dp, p0.data_ptr())
                d0 = eng.decide_fetch(nf)
                eng.decide_batch_dev(l1.data_ptr(), nf, ns, np.arange(nf, 2 * nf), flags, dp, p1.data_ptr())
                d1 = eng.decide_fetch(nf)
                eng.synchronize()
                assert torch.equal(l0.view(torch.int32), l1.view(torch.int32)), f"step {step}"
                assert d0.tobytes() == d1.tobytes(), f"step {step}: {d0} != {d1}"
                assert torch.equal(p0.view(torch.int32), p1.view(torch.int32)), f"step {step}"
        finally:
            eng.shard_comm_destroy()


def test_refusals_of_the_sharded_similarity_calls():
    import torch

    w = _world("binary")
    eng = _unsharded("binary", w)
    lst = w["lst"]
    ns, last, nf = len(lst), int(w["ids"].max()), 2
    ext = torch.cuda.ExternalStream(eng.stream)
    with torch.cuda.stream(ext):
        d_q = torch.from_numpy(w["q"][:nf].reshape(-1)).cuda()
        d_lst = torch.from_numpy(lst).cuda()
        d_rowids = torch.from_numpy(w["ids"]).cuda()
        d_tab = torch.from_numpy(w["table"]).cuda()
        d_fg = torch.from_numpy(w["gd_frames"][:nf]).cuda()
        d_words = torch.zeros(nf * F, dtype=torch.int32, device="cuda")
        pairs = torch.zeros(nf * ns, dtype=torch.int32, device="cuda")
        valid = torch.zeros(ns, dtype=torch.int32, device="cuda")
        like = torch.zeros(nf * ns, dtype=torch.float32, device="cuda")
        bad_rows = []
        for k, v in ((3, len(w["table"])), (4, -2)):
            r = w["row_of_k"].copy()
            r[k] = v
            bad_rows.append(torch.from_numpy(r).cuda())
        d_row = torch.from_numpy(w["row_of_k"]).cuda()

        def fused(**kw):
            eng.shard_localize_similarity_batch_dev(d_q.data_ptr(), nf, F, d_lst.data_ptr(), ns, d_rowids.data_ptr(), last, d_words.data_ptr(),
                                                    like.data_ptr(), **kw)

        def finalize(**kw):
            eng.shard_similarity_finalize_dev(pairs.data_ptr(), valid.data_ptr(), d_words.data_ptr(), nf, F, d_lst.data_ptr(), ns, like.data_ptr(),
                                              **kw)

        def code(fn, **kw):
            with pytest.raises(LcdError) as err:
                fn(**kw)
            return err.value.code

        gd = dict(d_frame_gdesc=d_fg.data_ptr(), d_map_gdesc=d_tab.data_ptr(), d_map_gdesc_row=d_row.data_ptr(), n_map_rows=len(w["table"]))
        assert code(fused) == LCD_ERR_STATE                                   # no communicator
        eng.shard_comm_init(Engine.shard_unique_id(), 0, 1)
        try:
            for fn in (fused, finalize):
                for r in bad_rows:
                    assert code(fn, **{**gd, "d_map_gdesc_row": r.data_ptr()}, dim=GD_DIM) == LCD_ERR_INVALID   # row outside the table
                for dim in (0, -4):
                    assert code(fn, **gd, dim=dim) == LCD_ERR_INVALID
                    assert code(fn, d_frame_gdesc=d_fg.data_ptr(), dim=dim) == LCD_ERR_INVALID
                assert code(fn, d_map_gdesc=d_tab.data_ptr(), n_map_rows=len(w["table"]), dim=GD_DIM) == LCD_ERR_INVALID  # table without rows
            assert code(eng.shard_localize_similarity_batch_dev, d_queries=d_q.data_ptr(), n_frames=1, nq=4097, d_sig_ids=d_lst.data_ptr(), ns=ns,
                        d_row_ids_global=d_rowids.data_ptr(), last_word_id=last, d_words_out=0, d_like_out=like.data_ptr()) == LCD_ERR_CAPACITY
            assert code(eng.shard_localize_similarity_batch_dev, d_queries=d_q.data_ptr(), n_frames=nf, nq=F, d_sig_ids=d_lst.data_ptr(), ns=ns,
                        d_row_ids_global=0, last_word_id=last, d_words_out=0, d_like_out=like.data_ptr()) == LCD_ERR_INVALID
            assert code(eng.shard_similarity_ids_dev, d_word_ids_all=d_words.data_ptr(), n_frames=nf, nq=F, d_sig_ids=d_lst.data_ptr(), ns=ns,
                        d_pairs_out=pairs.data_ptr(), d_valid_out=0) == LCD_ERR_INVALID
            fused(**gd, dim=GD_DIM)                                           # the good arguments pass after the refusals
            finalize(**gd, dim=GD_DIM)
            eng.synchronize()
        finally:
            eng.shard_comm_destroy()
    sharded = _engine("binary", w, w["ids"][3000:], w["vocab"][3000:], 3000)
    with pytest.raises(LcdError) as err:                                      # the unsharded group still refuses sharded engines
        sharded.localize_similarity_batch(w["q"][0], 1, lst)
    assert err.value.code == LCD_ERR_STATE
