"""Retrieval evaluation on the GPU (DESIGN 8): the ranks of the best positives against exact and fp64 brute force, symmetric tiles
against full tiles, the two-phase sharded form against the one call, the best positives and ranks against the layer's own
similarities, agreement with the layer's retrieval tops, and a set whose similarity matrix would not fit in HBM."""
import numpy as np
import pytest

from eval_ref import cuda, map_ref, planted

pytestmark = pytest.mark.gpu

PRECS = (0, 1, 2)          # capi.PREC_FP32_BF16X3, PREC_BF16, PREC_FP32_FP16X2


@pytest.mark.parametrize("prec", PRECS)
def test_exact_ranks_with_planted_ties(prec):
    from npairloss_b200 import capi
    rng = np.random.default_rng(20171225 + prec)
    # self-retrieval, ragged n and D
    n, D = 301, 37
    K, lab = planted(n, D, 60, rng)
    x = (K / 8.0).astype(np.float32)
    ev = capi.Evaluator(n, n, D, prec)
    xt, lt = cuda(x), cuda(lab)
    got = ev.rank(xt, lt, xt, lt, 0).cpu().numpy()
    want = map_ref(K @ K.T, lab, lab, 0)[3]
    assert (want > 1).sum() > 10 and (want == 0).sum() >= 5
    np.testing.assert_array_equal(got, want)
    ev.close()
    # query / gallery: disjoint sets, and queries that are a subset of the gallery
    nq, ng, D = 157, 389, 61
    Kg, lg = planted(ng, D, 50, rng)
    Kq = rng.integers(-8, 9, size=(nq, D)).astype(np.int64)
    Kq[: nq // 3] = Kg[rng.integers(0, ng, size=nq // 3)]           # exact duplicates of gallery rows
    lq = rng.integers(0, 50, size=nq).astype(np.float32)
    ev = capi.Evaluator(nq, ng, D, prec)
    qt, qlt, gt, glt = cuda((Kq / 8.0).astype(np.float32)), cuda(lq), cuda((Kg / 8.0).astype(np.float32)), cuda(lg)
    np.testing.assert_array_equal(ev.rank(qt, qlt, gt, glt, -1).cpu().numpy(), map_ref(Kq @ Kg.T, lq, lg, -1)[3])
    k = 101
    sub, subl = gt[k:k + nq].contiguous(), glt[k:k + nq].contiguous()
    np.testing.assert_array_equal(ev.rank(sub, subl, gt, glt, k).cpu().numpy(),
                                  map_ref(Kg[k:k + nq] @ Kg.T, lg[k:k + nq], lg, k)[3])
    ev.close()


@pytest.mark.parametrize("prec", (0, 2))
@pytest.mark.parametrize("D", (128, 512, 1024))
def test_ranks_within_fp64_bounds(prec, D):
    from npairloss_b200 import capi, synth
    n = 2000
    x, lab = synth.make_inputs(n, D, 20171226 + D, imgs_per_class=4, noise=1.5)
    xt, lt = cuda(x), cuda(lab)
    ev = capi.Evaluator(n, n, D, prec)
    rank = ev.rank(xt, lt, xt, lt, 0).cpu().numpy()
    ev.close()
    S = x.astype(np.float64) @ x.astype(np.float64).T
    np.fill_diagonal(S, -np.inf)
    same = lab[:, None] == lab[None, :]
    np.fill_diagonal(same, False)
    p = np.where(same, S, -np.inf).max(1)
    delta = 1e-5
    lo = 1 + (S > (p + delta)[:, None]).sum(1)        # the best positive always counts itself
    hi = (S >= (p - delta)[:, None]).sum(1)
    assert np.all(lo <= rank) and np.all(rank <= hi), np.nonzero((rank < lo) | (rank > hi))[0][:10]
    assert (lo != hi).mean() < 0.01


@pytest.mark.parametrize("prec", PRECS)
def test_symmetric_tiles_equal_full_tiles(prec):
    import torch
    from npairloss_b200 import capi, synth
    if capi.lib().npair_debug_mma_symmetric(prec) != 1:
        pytest.skip("this device's MMA is not bitwise symmetric in this operand format")
    n, D = 1000, 96
    x, lab = synth.make_inputs(n, D, 20171227, imgs_per_class=3, noise=2.0)
    xt, lt = cuda(x), cuda(lab)
    ev = capi.Evaluator(n, n, D, prec)
    r_sym = ev.rank(xt, lt, xt, lt, 0)
    r_full = ev.rank(xt, lt, xt.clone(), lt.clone(), 0)      # another buffer: every tile is computed
    torch.cuda.synchronize()
    assert torch.equal(r_sym, r_full)
    ev.close()


@pytest.mark.parametrize("prec", PRECS)
def test_sharded_gallery_equals_one_call(prec):
    import torch
    from npairloss_b200 import capi, synth
    n, D = 1100, 64
    x, lab = synth.make_inputs(n, D, 20171228, imgs_per_class=4, noise=2.0)
    xt, lt = cuda(x), cuda(lab)
    bounds = [0, 170, 777, n]                                  # three uneven shards
    ev = capi.Evaluator(n, n, D, prec)
    # the first 400 rows as queries against the rest (disjoint), and self-retrieval, whose one call computes only the tiles of the
    # upper triangle and mirrors them: the shards' full tiles give the same bits where the MMA is bitwise symmetric
    cases = [(xt[:400], lt[:400], xt[400:], lt[400:], -1)]
    if capi.lib().npair_debug_mma_symmetric(prec) == 1:
        cases.append((xt, lt, xt, lt, 0))
    for q, ql, g, gl, off in cases:
        q, ql, g, gl = q.contiguous(), ql.contiguous(), g.contiguous(), gl.contiguous()
        one = ev.rank(q, ql, g, gl, off)
        absmax = float(torch.maximum(q.abs().max(), g.abs().max()))
        cuts = [(a, min(b, g.shape[0])) for a, b in zip(bounds[:-1], bounds[1:]) if a < g.shape[0]]
        best = None
        for a, b in cuts:
            bp = ev.best_positive(q, ql, g[a:b].contiguous(), gl[a:b].contiguous(), absmax, off, a)
            best = bp if best is None else torch.maximum(best, bp)
        count = sum(ev.count(q, g[a:b].contiguous(), best, absmax, off, a).long() for a, b in cuts)
        torch.cuda.synchronize()
        assert torch.equal(count.int(), one), (off, (count.int() != one).sum().item())
    ev.close()


@pytest.mark.parametrize("prec", PRECS)
def test_sees_the_layers_similarities(prec):
    """The evaluator splits and pre-scales its operands exactly as the layer does: p* and the ranks taken from the layer's own fp32 S
    (world 1, S materialised) come out bit for bit.  Random unit rows at a ragged D, so every lo / mid piece is non-zero."""
    from npairloss_b200 import capi
    rng = np.random.default_rng(20171233 + prec)
    n, D = 1000, 100
    x = rng.standard_normal((n, D)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    lab = rng.integers(0, n // 3, size=n).astype(np.float32)           # about 3 rows per label, some without a positive
    xt, lt = cuda(x), cuda(lab)
    ctx = capi.Context(capi.make_config(n, D, sim_precision=prec))
    ctx.forward(xt, lt)
    S = ctx.debug_read(0, n * n).reshape(n, n)
    ctx.close()
    not_self = ~np.eye(n, dtype=bool)
    same = (lab[:, None] == lab[None, :]) & not_self
    p = np.where(same, S, np.float32(-np.inf)).max(1)
    want = np.where(p > -np.inf, ((S >= p[:, None]) & not_self).sum(1), 0)
    assert (p == -np.inf).sum() >= 5
    ev = capi.Evaluator(n, n, D, prec)
    best = ev.best_positive(xt, lt, xt, lt, float(np.abs(x).max()), 0).cpu().numpy()
    rank = ev.rank(xt, lt, xt, lt, 0).cpu().numpy()
    ev.close()
    np.testing.assert_array_equal(best.view(np.uint32), p.view(np.uint32))
    np.testing.assert_array_equal(rank, want)


def test_agrees_with_layer_tops():
    from npairloss_b200 import capi, synth
    from npairloss_b200.torch_api import recall_at_k
    Q, D = 2048, 128
    x, lab = synth.make_inputs(Q, D, 20171229, noise=1.5)
    xt, lt = cuda(x), cuda(lab)
    ctx = capi.Context(capi.make_config(Q, D))
    tops = ctx.forward(xt, lt)
    ctx.close()
    rec, rank = recall_at_k(xt, lt, ks=(1, 5, 10))
    assert rank.shape == (Q,) and int(rank.min()) >= 1
    for t, k in zip(tops[1:4], (1, 5, 10)):
        assert abs(rec[k] - t) * Q <= Q / 1000, (k, rec[k], t)


def test_recall_api_modes():
    import torch
    from npairloss_b200 import capi, synth
    from npairloss_b200.torch_api import recall_at_k
    x, lab = synth.make_inputs(600, 64, 20171231, imgs_per_class=3, noise=2.0)
    xt, lt = cuda(x), cuda(lab).long()
    rec, rank = recall_at_k(xt, lt)
    assert list(rec) == [1, 2, 4, 8] and all(0.0 <= v <= 1.0 for v in rec.values())
    assert rec[1] <= rec[2] <= rec[4] <= rec[8]
    # the same set passed as a gallery with every query its own row: the same ranks
    rec2, rank2 = recall_at_k(xt, lt, xt.clone(), lt.clone(), self_offset=0)
    if capi.lib().npair_debug_mma_symmetric(capi.PREC_FP32_FP16X2) == 1:
        assert torch.equal(rank, rank2) and rec2 == rec
    # disjoint: queries of classes that have gallery rows
    rec3, rank3 = recall_at_k(xt[:300], lt[:300], xt[300:], lt[300:])
    assert rank3.shape == (300,) and int(rank3.min()) >= 0


def test_batch_beyond_similarity_matrix():
    """Self-retrieval of B = 196608 at D = 128: the fp32 similarity matrix alone would take 155 GB."""
    import torch
    from npairloss_b200 import capi, synth
    B, D = 196608, 128
    x, lab = synth.make_inputs(B, D, 20171232, imgs_per_class=4, noise=1.5)
    xt, lt = cuda(x), cuda(lab)
    del x
    ws = capi.eval_workspace_bytes(B, B, D)
    capi.Evaluator(256, 256, D).close()                        # loads the module
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ev = capi.Evaluator(B, B, D)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    assert ws <= used <= ws + (256 << 20), (ws, used)
    rank = ev.rank(xt, lt, xt, lt, 0)
    torch.cuda.synchronize()
    ev.close()
    hits = int(((rank >= 1) & (rank <= 1)).sum())
    # chunked fp64 brute force of Recall@1
    xd = xt.double()
    ref = 0
    for a in range(0, B, 4096):
        S = xd[a:a + 4096] @ xd.T
        r = torch.arange(S.shape[0], device=S.device)
        S[r, a + r] = -float("inf")
        same = lt[a:a + 4096, None] == lt[None, :]
        same[r, a + r] = False
        p = torch.where(same, S, torch.full_like(S, -float("inf"))).max(1).values
        ref += int(((S >= p[:, None]).sum(1) == 1).logical_and(p > -float("inf")).sum())
        del S, same
    print(f"B={B}: Recall@1 {hits / B:.5f} (fp64 {ref / B:.5f}), workspace {ws / 1e6:.1f} MB, allocated {used / 1e6:.1f} MB")
    assert abs(hits - ref) <= B / 1000, (hits, ref)
