"""Cross-batch memory on the GPU (DESIGN 4.3): npair_forward_memory against npair_forward at m = 0, against the memory step of the
test reference on the GPU's own S, against the world-W external-collectives context it replaces, its independence of the capacity,
earlier calls and the memory buffers after the forward, its gradient, NPairLoss(memory_rows=M) and the refusals."""
import itertools

import numpy as np
import pytest

from npairloss_b200 import capi, synth
from gpu_harness import G_TOL
import sim_ref
from oracle import npair_oracle_np as onp

pytestmark = pytest.mark.gpu

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
PRECS = [FP16X2, BF16X3, BF16]
DEBUG = range(1, 10)
SPREAD = [dict(synth.DEFAULT_MINING), dict(synth.USAGE_MINING),
          dict(ap_region=0, ap_method=0, an_region=0, an_method=0, margin_diff=-0.02),
          dict(ap_region=1, ap_method=3, an_region=1, an_method=3, identsn=-0.4, diffsn=-0.3),
          dict(ap_region=1, ap_method=1, an_region=0, an_method=4, identsn=0.3, diffsn=-0.5, margin_ident=0.01)]


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _data(Q, m, D, seed, noise=0.7):
    """[x; x_mem] (Q + m unit rows) and their labels.  Classes of four rows, two in the batch and two among the memory rows: every
    anchor has a same-label row in the batch, and the memory shares classes with the batch as XBM's does.  Q even."""
    assert Q % 2 == 0
    k = max(Q, m) // 2 + 1
    x, lab = synth.make_inputs(4 * k, D, seed=seed, imgs_per_class=4, noise=noise)
    first = np.arange(4 * k) % 4 < 2
    rng = np.random.default_rng(seed)
    pb, pm = rng.permutation(Q), rng.permutation(2 * k)[:m]
    xb, lb, xm, lm = x[first][:Q][pb], lab[first][:Q][pb], x[~first][pm], lab[~first][pm]
    return np.ascontiguousarray(np.concatenate([xb, xm])), np.ascontiguousarray(np.concatenate([lb, lm]))


def _dev(torch, *arrs):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


def _ctx(Q, D, M, prec=FP16X2, mining=None, **extra):
    return capi.Context(capi.make_config(Q, D, sim_precision=prec, **(mining or {}), **extra), memory_rows=M)


def _step(torch, ctx, x, l, xm, lm, m, lw=1.0, S=True):
    """forward_memory + backward: dict(tops, dx, dbg[1..9], S [Q, Q + m])."""
    Q = x.shape[0]
    tops = np.array(ctx.forward_memory(x, l, xm, lm, m), dtype=np.float32)
    dx = torch.full_like(x, float("nan"))
    ctx.backward(lw, dx)
    torch.cuda.synchronize()
    out = dict(tops=tops, dx=dx.cpu().numpy(), dbg={w: ctx.debug_read(w, Q) for w in DEBUG})
    if S:
        out["S"] = ctx.debug_read(0, Q * (Q + m)).reshape(Q, Q + m)
    return out


def _same_bits(a, b, tag, S=True):
    np.testing.assert_array_equal(a["tops"].view(np.uint32), b["tops"].view(np.uint32), err_msg=f"{tag} tops")
    for w in DEBUG:
        np.testing.assert_array_equal(a["dbg"][w].view(np.uint32), b["dbg"][w].view(np.uint32), err_msg=f"{tag} debug {w}")
    np.testing.assert_array_equal(a["dx"].view(np.uint32), b["dx"].view(np.uint32), err_msg=f"{tag} gradient")
    if S and "S" in a and "S" in b:
        np.testing.assert_array_equal(a["S"].view(np.uint32), b["S"].view(np.uint32), err_msg=f"{tag} S")


def _check_parity(g, x, l, xm, lm, mining, prec, lw, num_tops=5, tag=""):
    """Level 1: S against fp64.  Level 2: the NumPy oracle's memory step (world 1 on [x; x_mem]) on the GPU's own S."""
    Q = x.shape[0]
    bad, m = sim_ref.check(g["S"], x, np.concatenate([x, xm]), prec)
    assert not bad, f"{tag} L1 S: {bad} ({m})"
    tops_o, dx_o, (st,) = onp.step_world_fp64(np.concatenate([x, xm]), np.concatenate([l, lm]), Q, 1, lw, S_inject_all=g["S"],
                                              num_tops=num_tops, **mining)
    tops_o, dx_o = tops_o[0], dx_o[:Q]
    np.testing.assert_array_equal(g["dbg"][1], st["posi_thr"], err_msg=f"{tag} posi_thr")
    np.testing.assert_array_equal(g["dbg"][2], st["nega_thr"], err_msg=f"{tag} nega_thr")
    np.testing.assert_allclose(g["tops"][0], tops_o[0], rtol=1e-5, atol=1e-6, err_msg=f"{tag} loss")
    n_ret = max(0, num_tops - 2)
    if n_ret:
        d = np.abs(g["tops"][1:1 + n_ret] - tops_o[1:1 + n_ret]) * Q
        assert d.max() <= max(1.0, Q / 1000.0) + 1e-3, f"{tag} retrieval counters differ by {d.max()} rows"
    np.testing.assert_allclose(g["tops"][num_tops - 1], tops_o[num_tops - 1], rtol=2e-6, err_msg=f"{tag} asum")
    assert np.isfinite(g["dx"]).all(), f"{tag} non-finite gradient"
    gn = max(float(np.linalg.norm(dx_o)), 1e-20)
    ge = float(np.linalg.norm(g["dx"] - dx_o))
    assert ge <= G_TOL[prec] * gn, f"{tag} gradient normwise error {ge / gn:.3e}"


# ---------------------------------------------------------------------------------------------------------- 1. m = 0
@pytest.mark.parametrize("prec", PRECS)
def test_no_memory_rows_is_npair_forward_bit_for_bit(torch, prec):
    """On a memory context, m = 0 -- also right after a call with m = M -- is npair_forward of a plain context."""
    Q, D, M = 200, 72, 300
    x, l = _data(Q, M, D, 3)
    xt, lt, xmt, lmt = _dev(torch, x[:Q], l[:Q], x[Q:], l[Q:])
    for k, mining in enumerate(SPREAD):
        plain = capi.Context(capi.make_config(Q, D, sim_precision=prec, **mining))
        mem = _ctx(Q, D, M, prec, mining)
        try:
            tops = np.array(plain.forward(xt, lt), dtype=np.float32)
            dx = torch.full_like(xt, float("nan"))
            plain.backward(0.8, dx)
            torch.cuda.synchronize()
            ref = dict(tops=tops, dx=dx.cpu().numpy(), dbg={w: plain.debug_read(w, Q) for w in DEBUG}, S=plain.debug_read(0, Q * Q).reshape(Q, Q))
            _step(torch, mem, xt, lt, xmt, lmt, M, 0.8, S=False)
            _same_bits(_step(torch, mem, xt, lt, None, None, 0, 0.8), ref, f"prec {prec} mining {k}")
        finally:
            plain.close(); mem.close()


# ---------------------------------------------------------------------------------------------------------- 2. L2 parity
@pytest.mark.parametrize("fused", [True, False])
def test_l2_parity_every_mining_combination(torch, fused):
    """All 100 (region, method)^2 combinations at ragged Q, D and m, memory sharing classes with the batch."""
    Q, D = 44, 36
    ms = [1, 37, Q, 3 * Q + 5]
    M = max(ms)
    x, l = _data(Q, M, D, 17)
    xt, lt, xmt, lmt = _dev(torch, x[:Q], l[:Q], x[Q:], l[Q:])
    flags = 0 if fused else capi.FLAG_NO_FUSED_GRAD
    for apR, apM, anR, anM in itertools.product([0, 1], range(5), [0, 1], range(5)):
        mining = dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3, ap_region=apR, ap_method=apM, an_region=anR,
                      an_method=anM)
        ctx = _ctx(Q, D, M, FP16X2, mining, flags=flags)
        try:
            for m in ms:
                g = _step(torch, ctx, xt, lt, xmt, lmt, m, 0.7)
                _check_parity(g, x[:Q], l[:Q], x[Q:Q + m], l[Q:Q + m], mining, FP16X2, 0.7, tag=f"fused {fused} {apR}{apM}{anR}{anM} m {m}")
        finally:
            ctx.close()


@pytest.mark.parametrize("prec", [BF16X3, BF16])
def test_l2_parity_other_formats(torch, prec):
    Q, D, m = 70, 50, 131
    x, l = _data(Q, m, D, 23)
    xt, lt, xmt, lmt = _dev(torch, x[:Q], l[:Q], x[Q:], l[Q:])
    for fused in (True, False):
        for mining in SPREAD:
            ctx = _ctx(Q, D, m, prec, mining, flags=0 if fused else capi.FLAG_NO_FUSED_GRAD)
            try:
                g = _step(torch, ctx, xt, lt, xmt, lmt, m, 1.0)
                _check_parity(g, x[:Q], l[:Q], x[Q:], l[Q:], mining, prec, 1.0, tag=f"prec {prec} fused {fused} {mining}")
            finally:
                ctx.close()


# ---------------------------------------------------------------------------------------------------------- 3. workaround
@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("mining", [synth.USAGE_MINING, dict(ap_region=0, ap_method=3, identsn=-0.4, an_region=0, an_method=4, diffsn=-0.3)])
def test_equals_the_world_w_external_collectives_workaround(torch, W, mining):
    """m = (W - 1) Q: the forward is rank 0 of a world-W external-collectives context on [x; x_mem] bit for bit, and the gradient is
    that context's d_local_half + W d_total_half[:Q]."""
    Q, D = 96, 64
    m = (W - 1) * Q
    x, l = _data(Q, m, D, 40 + W)
    xt_all, lt_all = _dev(torch, x, l)
    mem = _ctx(Q, D, m, FP16X2, mining)
    ext = capi.Context(capi.make_config(Q, D, world=W, rank=0, bwd_exchange=1, **mining))
    try:
        g = _step(torch, mem, xt_all[:Q].contiguous(), lt_all[:Q].contiguous(), xt_all[Q:].contiguous(), lt_all[Q:].contiguous(), m, 1.3)
        tops = np.array(ext.forward_gathered(xt_all, lt_all), dtype=np.float32)
        lh = torch.full((Q, D), float("nan"), device="cuda")
        th = torch.full((Q + m, D), float("nan"), device="cuda")
        ext.backward_partial(1.3, lh, th)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(g["tops"].view(np.uint32), tops.view(np.uint32))
        for w in DEBUG:
            np.testing.assert_array_equal(g["dbg"][w].view(np.uint32), ext.debug_read(w, Q).view(np.uint32), err_msg=f"debug {w}")
        np.testing.assert_array_equal(g["S"].view(np.uint32), ext.debug_read(0, Q * (Q + m)).reshape(Q, Q + m).view(np.uint32))
        ref = (lh + W * th[:Q]).cpu().numpy()
        assert np.linalg.norm(g["dx"] - ref) <= 1e-5 * np.linalg.norm(ref)
    finally:
        mem.close(); ext.close()


# ---------------------------------------------------------------------------------------------------------- 4. independence
@pytest.mark.parametrize("prec", [FP16X2, BF16X3])
@pytest.mark.parametrize("fused", [True, False])
def test_results_do_not_depend_on_capacity_or_earlier_calls(torch, prec, fused):
    Q, D, M, m2 = 130, 40, 900, 261
    mining = dict(synth.USAGE_MINING)
    flags = 0 if fused else capi.FLAG_NO_FUSED_GRAD
    x, l = _data(Q, M, D, 51)
    big = x[Q:].copy()
    big[::7] *= 1000.0                                  # a large pre-scale and large similarities in the first call
    xt, lt, bigt, lmt = _dev(torch, x[:Q], l[:Q], big, l[Q:])
    xm2, lm2 = _dev(torch, x[Q:Q + m2], l[Q:Q + m2])
    used = _ctx(Q, D, M, prec, mining, flags=flags)
    fresh = _ctx(Q, D, m2, prec, mining, flags=flags)
    try:
        _step(torch, used, xt, lt, bigt, lmt, M, 1.0, S=False)
        a = _step(torch, used, xt, lt, xm2, lm2, m2, 1.0)
        b = _step(torch, fresh, xt, lt, xm2, lm2, m2, 1.0)
        _same_bits(a, b, "capacity")
        _same_bits(_step(torch, used, xt, lt, xm2, lm2, m2, 1.0), a, "repeat")
    finally:
        used.close(); fresh.close()


def _splits(Q, D, N, fused, sms):
    """The gradient's split-K count at N database columns (host.cuh split_k; fp16x2: 32-column K blocks on both gradient paths)."""
    kb, tiles, min_kb = (N + 31) // 32, ((Q + 127) // 128) * ((D + 255) // 256), 8 if fused else 4
    s = max(1, min(16, sms // tiles, kb // min_kb))
    kpb = (kb + s - 1) // s
    return (kb + kpb - 1) // kpb


@pytest.mark.parametrize("Q,D,M,m,fused", [(512, 512, 2049, 2048, True), (1024, 128, 1, 0, False), (512, 512, 4113, 4096, True)])
def test_a_smaller_m_with_more_split_k_slices(torch, Q, D, M, m, fused):
    """The split-K count is not monotone in N (its empty splits are dropped): at these shapes m gets more slices than the capacity M.
    The call must still equal a fresh context of capacity m bit for bit."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if _splits(Q, D, Q + m, fused, sms) <= _splits(Q, D, Q + M, fused, sms):
        pytest.skip(f"{sms} SMs: m = {m} takes no more split-K slices than M = {M}")
    x, l = _data(Q, M, D, 141)
    xt, lt, xm, lm = _dev(torch, x[:Q], l[:Q], x[Q:], l[Q:])
    flags = 0 if fused else capi.FLAG_NO_FUSED_GRAD
    used = _ctx(Q, D, M, FP16X2, synth.USAGE_MINING, flags=flags)
    fresh = _ctx(Q, D, m, FP16X2, synth.USAGE_MINING, flags=flags)
    try:
        _step(torch, used, xt, lt, xm, lm, M, 1.0, S=False)
        a = _step(torch, used, xt, lt, xm, lm, m, 1.0)
        b = _step(torch, fresh, xt, lt, xm, lm, m, 1.0)
        _same_bits(a, b, f"Q {Q} D {D} M {M} m {m}")
    finally:
        used.close(); fresh.close()


def test_memory_rows_may_be_overwritten_after_the_forward(torch):
    Q, D, m = 100, 48, 333
    x, l = _data(Q, m, D, 61)
    xt, lt = _dev(torch, x[:Q], l[:Q])
    for fused in (True, False):
        ctx = _ctx(Q, D, m, FP16X2, synth.USAGE_MINING, flags=0 if fused else capi.FLAG_NO_FUSED_GRAD)
        try:
            xm, lm = _dev(torch, x[Q:], l[Q:])
            ref = _step(torch, ctx, xt, lt, xm, lm, m, 1.0)
            ctx.forward_memory(xt, lt, xm, lm, m)
            xm.fill_(float("nan")); lm.fill_(float("nan"))          # in stream order, before the backward
            dx = torch.full_like(xt, float("nan"))
            ctx.backward(1.0, dx)
            torch.cuda.synchronize()
            np.testing.assert_array_equal(dx.cpu().numpy().view(np.uint32), ref["dx"].view(np.uint32))
        finally:
            ctx.close()


# ---------------------------------------------------------------------------------------------------------- 5. gradient
def test_true_gradient_matches_finite_differences(torch):
    """RAND mining (no thresholds: the loss is smooth); 2 x the backward is the gradient of the loss with the memory held fixed."""
    from npairloss_b200.torch_api import NPairLoss
    Q, D, m = 24, 16, 40
    x, l = _data(Q, m, D, 71, noise=1.5)
    xt, lt, xm, lm = _dev(torch, x[:Q], l[:Q], x[Q:], l[Q:])
    ctx = _ctx(Q, D, m, BF16X3, synth.DEFAULT_MINING)
    try:
        ctx.forward_memory(xt, lt, xm, lm, m)
        g = torch.empty_like(xt)
        ctx.backward(1.0, g)
        g = 2.0 * g.double().cpu().numpy()
        rng = np.random.default_rng(3)
        for _ in range(4):
            v = rng.standard_normal((Q, D)).astype(np.float32)
            v /= np.linalg.norm(v)
            eps = 2e-2
            lp = ctx.forward_memory(xt + eps * torch.from_numpy(v).cuda(), lt, xm, lm, m)[0]
            lmn = ctx.forward_memory(xt - eps * torch.from_numpy(v).cuda(), lt, xm, lm, m)[0]
            fd = (lp - lmn) / (2 * eps)
            an = float((g * v).sum())
            assert abs(fd - an) <= 2e-2 * abs(an) + 2e-4, (fd, an)
    finally:
        ctx.close()
    assert NPairLoss(memory_rows=8, true_gradient=True)._mem_cap == 8


def test_normalize_input_with_a_memory(torch, oracle):
    Q, D, m = 64, 40, 150
    x, l = _data(Q, m, D, 81)
    raw = x[:Q] * np.linspace(0.5, 3.0, Q, dtype=np.float32)[:, None]
    xt, lt, xm, lm = _dev(torch, raw, l[:Q], x[Q:], l[Q:])
    for fused in (True, False):
        ctx = _ctx(Q, D, m, FP16X2, synth.USAGE_MINING, normalize_input=1, flags=0 if fused else capi.FLAG_NO_FUSED_GRAD)
        try:
            g = _step(torch, ctx, xt, lt, xm, lm, m, 1.0)
        finally:
            ctx.close()
        y, inv = oracle.l2normalize_forward(raw)
        tops_o, dy, (st,) = onp.step_world_fp64(np.concatenate([y, x[Q:]]), l, Q, 1, 1.0, S_inject_all=g["S"], **synth.USAGE_MINING)
        tops_o, dy = tops_o[0], dy[:Q]
        np.testing.assert_allclose(g["tops"][0], tops_o[0], rtol=1e-5, atol=1e-6)
        np.testing.assert_array_equal(g["dbg"][1], st["posi_thr"])
        dx_o = oracle.l2normalize_backward(y, inv, dy.astype(np.float32))
        assert np.linalg.norm(g["dx"] - dx_o) <= 1e-5 * np.linalg.norm(dx_o)


def test_unaligned_memory_pointers(torch):
    """Memory rows and labels that start 4 bytes past an allocation give the same bits (D odd: the rows themselves are unaligned too)."""
    Q, D, m = 90, 33, 170
    x, l = _data(Q, m, D, 91)
    xt, lt = _dev(torch, x[:Q], l[:Q])
    xm, lm = _dev(torch, x[Q:], l[Q:])
    xm_buf = torch.empty(m * D + 1, device="cuda"); xm_buf[1:].copy_(xm.reshape(-1))
    lm_buf = torch.empty(m + 1, device="cuda"); lm_buf[1:].copy_(lm)
    st = torch.cuda.current_stream().cuda_stream
    ctx = _ctx(Q, D, m, FP16X2, synth.USAGE_MINING)
    try:
        ref = _step(torch, ctx, xt, lt, xm, lm, m, 1.0)
        tops = np.array(ctx.forward_memory_ptr(xt.data_ptr(), lt.data_ptr(), xm_buf.data_ptr() + 4, lm_buf.data_ptr() + 4, m, st),
                        dtype=np.float32)
        dx = torch.full_like(xt, float("nan"))
        ctx.backward(1.0, dx)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(tops.view(np.uint32), ref["tops"].view(np.uint32))
        np.testing.assert_array_equal(dx.cpu().numpy().view(np.uint32), ref["dx"].view(np.uint32))
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------- 6. NPairLoss
def test_npairloss_memory_ring(torch):
    from npairloss_b200.torch_api import NPairLoss
    Q, D, M, steps = 32, 24, 96, 6
    mining = dict(synth.USAGE_MINING)
    x, l = synth.make_inputs(Q * steps, D, seed=101, noise=0.7)
    batches = [_dev(torch, x[t * Q:(t + 1) * Q], l[t * Q:(t + 1) * Q]) for t in range(steps)]
    fn = NPairLoss(memory_rows=M, **mining)
    direct = _ctx(Q, D, M, FP16X2, mining)
    try:
        for t, (xb, lb) in enumerate(batches):
            mx, ml = fn.memory()
            mx = None if mx is None else mx.clone()
            ml = None if ml is None else ml.clone()
            m = 0 if mx is None else mx.shape[0]
            assert m == min(t * Q, M)
            feat = xb.clone().requires_grad_(True)
            loss, tops = fn(feat, lb)
            loss.backward()
            want = direct.forward_memory(xb, lb, mx, ml, m)
            dx = torch.empty_like(xb)
            direct.backward(1.0, dx)
            torch.cuda.synchronize()
            assert np.float32(loss.item()).view(np.uint32) == np.float32(want[0]).view(np.uint32), t
            assert torch.equal(feat.grad, dx), t
            # the ring after step t: batch b in slots (b Q) mod M for the last M / Q batches
            rx, rl = fn.memory()
            assert not rx.requires_grad
            for b in range(max(0, t + 1 - M // Q), t + 1):
                s = (b * Q) % M
                assert torch.equal(rx[s:s + Q], batches[b][0]) and torch.equal(rl[s:s + Q], batches[b][1]), (t, b)
        fn.reset_memory()
        assert fn.memory()[0].shape[0] == 0
        loss_r, _ = fn(batches[0][0], batches[0][1])
        loss_p, _ = NPairLoss(**mining)(batches[0][0], batches[0][1])
        assert np.float32(loss_r.item()).view(np.uint32) == np.float32(loss_p.item()).view(np.uint32)
        # a second forward through the module before the first one's backward is refused
        f1 = batches[1][0].clone().requires_grad_(True)
        l1, _ = fn(f1, batches[1][1])
        fn(batches[2][0], batches[2][1])
        with pytest.raises(RuntimeError):
            l1.backward()
    finally:
        direct.close()


def test_npairloss_memory_survives_a_new_batch_size_and_normalises(torch):
    from npairloss_b200.torch_api import NPairLoss
    D, M = 20, 70
    x, l = _data(70, 0, D, 111)
    raw = x * 3.0
    fn = NPairLoss(memory_rows=M, normalize_input=1)
    a = _dev(torch, raw[:40], l[:40])
    b = _dev(torch, raw[40:70], l[40:70])
    fn(*a)
    fn(*b)                                               # a new Q re-creates the context, the ring keeps its rows
    rx, _ = fn.memory()
    assert rx.shape[0] == 70
    y, _ = capi.l2normalize_forward(a[0])
    assert torch.equal(rx[:40], y)
    with pytest.raises(ValueError):
        NPairLoss(world=2, memory_rows=M)


# ---------------------------------------------------------------------------------------------------------- 7. refusals
def test_refusals_enqueue_nothing(torch):
    Q, D, M = 64, 32, 128
    for kw in (dict(world=2), dict(sim_block_rows=128, Q=256), dict(gemm_backend=capi.GEMM_SIMT_CHECK), dict(global_scope=1)):
        q = kw.pop("Q", Q)
        with pytest.raises(capi.NpairError) as e:
            capi.Context(capi.make_config(q, D, **kw), memory_rows=M)
        assert e.value.code == -1, kw
    x, l = _data(Q, M + 1, D, 121)
    xt, lt, xm, lm = _dev(torch, x[:Q], l[:Q], x[Q:], l[Q:])
    st = torch.cuda.current_stream().cuda_stream
    ctx = _ctx(Q, D, M)
    plain = {k: capi.Context(capi.make_config(Q, D, **kw)) for k, kw in
             (("simt", dict(gemm_backend=capi.GEMM_SIMT_CHECK)), ("plain", dict()))}
    try:
        torch.cuda.synchronize()
        n0 = capi.kernel_launches()
        for c, args in ((ctx, (xm.data_ptr(), lm.data_ptr(), M + 1)), (ctx, (xm.data_ptr(), lm.data_ptr(), -1)),
                        (ctx, (None, lm.data_ptr(), 5)), (ctx, (xm.data_ptr(), None, 5)),
                        (plain["plain"], (xm.data_ptr(), lm.data_ptr(), 1)), (plain["simt"], (None, None, 0))):
            with pytest.raises(capi.NpairError) as e:
                c.forward_memory_ptr(xt.data_ptr(), lt.data_ptr(), *args, stream=st)
            assert e.value.code == -1, args
        assert capi.kernel_launches() == n0
        ctx.forward_memory(xt, lt, xm, lm, M)                # the context is still usable
    finally:
        ctx.close()
        for c in plain.values():
            c.close()


# ---------------------------------------------------------------------------------------------------------- 8. larger case
@pytest.mark.parametrize("mining", [dict(ap_region=1, ap_method=3, identsn=-0.4, an_region=1, an_method=3, diffsn=-0.3, margin_diff=-0.02),
                                    dict(ap_region=0, ap_method=0, an_region=0, an_method=0, margin_diff=-0.05)])
def test_larger_case(torch, mining):
    Q, D, m = 1024, 128, 16384
    x, l = _data(Q, m, D, 131, noise=1.5)
    xt, lt, xm, lm = _dev(torch, x[:Q], l[:Q], x[Q:], l[Q:])
    ctx = _ctx(Q, D, m, FP16X2, mining)
    try:
        g = _step(torch, ctx, xt, lt, xm, lm, m, 1.0)
    finally:
        ctx.close()
    _check_parity(g, x[:Q], l[:Q], x[Q:], l[Q:], mining, FP16X2, 1.0, tag=str(mining))
