"""The memory rows' gradient on the GPU (DESIGN 4.6): npair_backward_memory's anchor gradient against npair_backward bit for bit, its
identities (m = 0, device weight, unit anchor weights, repeat runs, capacity and earlier calls), the memory-row gradient against the
fp64 step of grad_ref on the GPU's own S (normwise and by its fp64 rules), against the world-W external-collectives workaround, the
refusals, graph capture, and NPairLoss(extra_rows=...) with learnable proxies."""
import ctypes as C
import itertools

import numpy as np
import pytest

import grad_ref
from gpu_harness import G_TOL
from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
USAGE = dict(synth.USAGE_MINING)
ALL_MINING = [dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3, ap_region=apR, ap_method=apM, an_region=anR,
                   an_method=anM)
              for apR, apM, anR, anM in itertools.product([0, 1], [0, 1, 2, 3, 4], [0, 1], [0, 1, 2, 3, 4])]


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _data(Q, m, D, seed, noise=0.7, classes=None):
    """Q anchors and m memory rows (unit rows); the memory rows' labels fall into the anchors' classes, as proxies' do.  Every anchor
    has a same-label anchor (odd Q: the last one joins the pair before it)."""
    x, lab = synth.make_inputs(Q + m, D, seed=seed, imgs_per_class=2, noise=noise)
    lab = lab.copy()
    if Q % 2 and Q > 1:
        lab[Q - 1] = lab[Q - 2]
    ncls = classes or max(1, Q // 2)
    lab[Q:] = np.random.default_rng(seed).integers(0, ncls + 3, m).astype(np.float32)     # a few classes no anchor has
    return x[:Q].copy(), lab[:Q].copy(), x[Q:].copy(), lab[Q:].copy()


def _dev(torch, *arrs):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


def _ctx(Q, D, M, prec=FP16X2, mining=None, **extra):
    return capi.Context(capi.make_config(Q, D, sim_precision=prec, **(mining or {}), **extra), memory_rows=M)


def _mem_splits(Q, D, m):
    """The memory-row gradient's split-K count (ctx.cu mem_grad_split, host.cuh split_k): an m x D output of 128 x 256 tiles over
    ceil(Q / 32) K blocks, at least 8 per split, at most 16 splits, at most one tile per SM."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kb, tiles = (Q + 31) // 32, ((m + 127) // 128) * ((D + 255) // 256)
    s = max(1, min(16, sms // tiles, kb // 8))
    kpb = (kb + s - 1) // s
    return (kb + kpb - 1) // kpb


def _mem_ref(x, l, y, ly, S, w=None, loss_weight=1.0, **mining):
    """R, B and R32 of the memory rows: rows [Q, N) of grad_ref.step over the database [x; y]."""
    Q = x.shape[0]
    ref = grad_ref.step(np.concatenate([x, y]), np.concatenate([l, ly]), Q, 1, S, w, loss_weight, **mining)
    return {k: ref[k][Q:] for k in ("R", "B", "R32")}


def _bits(a):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _mem_step(torch, ctx, x, l, y, ly, lw=1.0, device_weight=False, S=False):
    """forward_memory + backward_memory: (dx, d_mem[, S]) as host arrays."""
    Q, m = x.shape[0], y.shape[0]
    ctx.forward_memory(x, l, y, ly, m)
    dx = torch.full_like(x, float("nan"))
    dm = torch.full((max(m, 1), x.shape[1]), float("nan"), device="cuda")
    if device_weight:
        ctx.backward_memory_device_weight(torch.full((1,), lw, device="cuda"), dx, dm)
    else:
        ctx.backward_memory(lw, dx, dm)
    torch.cuda.synchronize()
    out = [dx.cpu().numpy(), dm[:m].cpu().numpy()]
    if S:
        out.append(ctx.debug_read(0, Q * (Q + m)).reshape(Q, Q + m))
    return out


# ---------------------------------------------------------------------------------------------------------- 1. identities
@pytest.mark.parametrize("prec", [FP16X2, BF16X3, BF16])
@pytest.mark.parametrize("normalize", [0, 1])
def test_anchor_gradient_is_npair_backward_and_runs_repeat(torch, prec, normalize):
    """The anchor gradient has the bits of npair_backward after the same forward; the device loss weight gives the host weight's bits;
    two runs give the same bits."""
    Q, D, m = 258, 136, 301
    x, l, y, ly = _data(Q, m, D, 11, noise=2.0)
    xt, lt, yt, lyt = _dev(torch, x, l, y, ly)
    ctx = _ctx(Q, D, m, prec, USAGE, normalize_input=normalize)
    try:
        ctx.forward_memory(xt, lt, yt, lyt, m)
        ref = torch.full_like(xt, float("nan"))
        ctx.backward(0.75, ref)
        dx, dm = _mem_step(torch, ctx, xt, lt, yt, lyt, 0.75)
        np.testing.assert_array_equal(_bits(dx), _bits(ref), err_msg="anchor gradient")
        assert np.isfinite(dm).all() and np.abs(dm).max() > 0
        dx2, dm2 = _mem_step(torch, ctx, xt, lt, yt, lyt, 0.75, device_weight=True)
        np.testing.assert_array_equal(_bits(dx2), _bits(dx), err_msg="device weight: anchors")
        np.testing.assert_array_equal(_bits(dm2), _bits(dm), err_msg="device weight: memory rows")
        dx3, dm3 = _mem_step(torch, ctx, xt, lt, yt, lyt, 0.75)
        np.testing.assert_array_equal(_bits(dx3), _bits(dx), err_msg="second run: anchors")
        np.testing.assert_array_equal(_bits(dm3), _bits(dm), err_msg="second run: memory rows")
    finally:
        ctx.close()


def test_no_memory_rows_leaves_the_output_untouched(torch):
    Q, D = 128, 64
    x, l, _, _ = _data(Q, 0, D, 13)
    xt, lt = _dev(torch, x, l)
    ctx = _ctx(Q, D, 64)
    try:
        ctx.forward_memory(xt, lt, None, None, 0)
        ref = torch.empty_like(xt)
        ctx.backward(1.0, ref)
        dx, dm = torch.empty_like(xt), torch.full((64, D), float("nan"), device="cuda")
        ctx.backward_memory(1.0, dx, dm)
        torch.cuda.synchronize()
        assert torch.isnan(dm).all()
        np.testing.assert_array_equal(_bits(dx), _bits(ref))
    finally:
        ctx.close()


def test_unit_anchor_weights_are_no_weights(torch):
    Q, D, m = 200, 96, 150
    x, l, y, ly = _data(Q, m, D, 17)
    xt, lt, yt, lyt = _dev(torch, x, l, y, ly)
    ctx = _ctx(Q, D, m, FP16X2, USAGE)
    try:
        plain = _mem_step(torch, ctx, xt, lt, yt, lyt)
        ctx.set_anchor_io(torch.ones(Q, device="cuda"), None)
        weighted = _mem_step(torch, ctx, xt, lt, yt, lyt)
        ctx.set_anchor_io(None, None)
        for a, b, tag in zip(plain, weighted, ("anchors", "memory rows")):
            np.testing.assert_array_equal(_bits(a), _bits(b), err_msg=tag)
    finally:
        ctx.close()


@pytest.mark.parametrize("prec", [FP16X2, BF16X3])
@pytest.mark.parametrize("Q,D,ms,split", [(130, 72, (261, 37), False), (514, 200, (100, 37, 1), True), (1030, 136, (100, 37), True)])
def test_results_do_not_depend_on_capacity_or_earlier_calls(torch, prec, Q, D, ms, split):
    """A context of capacity 3000 after a call with m = 3000 (large rows: another pre-scale) gives, at each m of `ms`, the bits of a
    context made for exactly that m.  split: the memory gradient cuts K into several slices at each of those m (asserted), through a
    partial buffer that the two contexts size for different capacities."""
    M = 3000
    if split:
        assert all(_mem_splits(Q, D, m) > 1 for m in ms), [_mem_splits(Q, D, m) for m in ms]
    else:
        assert all(_mem_splits(Q, D, m) == 1 for m in ms)
    x, l, y, ly = _data(Q, M, D, 19)
    big = y.copy()
    big[::5] *= 1000.0
    xt, lt, bigt, lyt = _dev(torch, x, l, big, ly)
    used = _ctx(Q, D, M, prec, USAGE)
    try:
        _mem_step(torch, used, xt, lt, bigt, lyt)
        for m in ms:
            yt, lmt = _dev(torch, y[:m], ly[:m])
            fresh = _ctx(Q, D, m, prec, USAGE)
            try:
                a, b = _mem_step(torch, used, xt, lt, yt, lmt), _mem_step(torch, fresh, xt, lt, yt, lmt)
            finally:
                fresh.close()
            for u, v, tag in zip(a, b, ("anchors", "memory rows")):
                np.testing.assert_array_equal(_bits(u), _bits(v), err_msg=f"m = {m} {tag}")
    finally:
        used.close()


# ---------------------------------------------------------------------------------------------------------- 2. L2 parity
@pytest.mark.parametrize("Q,m", [(130, 1), (130, 37), (130, 261), (129, 37), (131, 261), (514, 37), (1030, 100), (1027, 1)])
def test_l2_parity_every_mining_combination(torch, Q, m):
    """On the GPU's own S, d_mem_diff is within 1e-5 normwise of the reference for all 100 mining combinations, D = 200, with anchor
    weights with zeros and NaN labels among the memory rows.  Q is no multiple of 128 and covers every remainder Q & 3 of the transposed
    tile's column offset (130, 514: 2; 129: 1; 131, 1027: 3; 1030: 2); from Q = 514 on the memory gradient splits K (asserted)."""
    D = 200
    assert (_mem_splits(Q, D, m) > 1) == (Q > 480), _mem_splits(Q, D, m)
    x, l, y, ly = _data(Q, m, D, 23 + m + Q, noise=1.2)
    ly[::9] = np.nan
    rng = np.random.default_rng(m)
    w = rng.uniform(0, 1, Q).astype(np.float32)
    w[::7] = 0.0
    w[1::11] = 1.0
    xt, lt, yt, lyt, wt = _dev(torch, x, l, y, ly, w)
    worst = 0.0
    for i, mining in enumerate(ALL_MINING):
        ctx = _ctx(Q, D, m, FP16X2, mining)
        try:
            if i % 2:
                ctx.set_anchor_io(wt, None)
            _, dm, S = _mem_step(torch, ctx, xt, lt, yt, lyt, 1.3, S=True)
        finally:
            ctx.close()
        ref = _mem_ref(x, l, y, ly, S, w if i % 2 else None, 1.3, **mining)["R"]
        err = float(np.linalg.norm(dm - ref))
        assert err <= 1e-5 * max(float(np.linalg.norm(ref)), 1e-30), f"{mining} weighted {bool(i % 2)}: {err / np.linalg.norm(ref):.3e}"
        worst = max(worst, err / max(float(np.linalg.norm(ref)), 1e-30))
    print(f"Q = {Q}, m = {m}, {_mem_splits(Q, D, m)} split(s): worst normwise error {worst:.2e}")


@pytest.mark.parametrize("prec", [BF16X3, BF16])
def test_l2_parity_other_formats(torch, prec):
    Q, D, m = 130, 200, 261
    x, l, y, ly = _data(Q, m, D, 29, noise=1.2)
    xt, lt, yt, lyt = _dev(torch, x, l, y, ly)
    for mining in ALL_MINING[::9]:
        ctx = _ctx(Q, D, m, prec, mining)
        try:
            _, dm, S = _mem_step(torch, ctx, xt, lt, yt, lyt, S=True)
        finally:
            ctx.close()
        ref = _mem_ref(x, l, y, ly, S, **mining)["R"]
        assert np.linalg.norm(dm - ref) <= G_TOL[prec] * max(np.linalg.norm(ref), 1e-30), mining


# ---------------------------------------------------------------------------------------------------------- 3. fp64 rules
@pytest.mark.parametrize("kind,Q,m,D", [("cone", 512, 16384, 128), ("cone", 384, 1000, 96), ("spread", 384, 2000, 512)])
def test_fp64_rules(torch, kind, Q, m, D):
    """grad_ref.violations of d_mem_diff against the fp64 product of the step's weights on the GPU's S: the fused path's componentwise
    bound over an accumulation of Q columns, and the normwise and per-row rules."""
    if kind == "cone":
        xa, la = grad_ref.cone_inputs(Q + m, D, 0.1, 31)
        la = np.concatenate([la[:Q], la[Q:] % (Q // 2)]).astype(np.float32)
        x, l, y, ly = xa[:Q], la[:Q], xa[Q:], la[Q:]
    else:
        x, l, y, ly = _data(Q, m, D, 37, noise=2.5)
    xt, lt, yt, lyt = _dev(torch, x, l, y, ly)
    ctx = _ctx(Q, D, m, FP16X2, USAGE, num_tops=2)
    try:
        _, dm, S = _mem_step(torch, ctx, xt, lt, yt, lyt, S=True)
    finally:
        ctx.close()
    ref = _mem_ref(x, l, y, ly, S, **USAGE)
    k = grad_ref.SGEMM_FACTOR["accumulator" if kind == "cone" else "spread"]
    bad, meas = grad_ref.violations(dm, ref, grad_ref.tau(FP16X2, "fused", Q), rel=G_TOL[FP16X2], k_sgemm=k)
    print(f"{kind} Q {Q} m {m}: normwise {meas['normwise']:.2e} (sgemm {meas['sgemm']:.2e}) worst row {meas['row']:.3f}, "
          f"componentwise {meas['comp']:.1f} x 2^-24 of B")
    assert not bad, "; ".join(bad)


# ---------------------------------------------------------------------------------------------------------- 4. the workaround
@pytest.mark.parametrize("W", [2, 3])
def test_equals_the_world_w_external_collectives_workaround(torch, W):
    """m = (W - 1) Q: d_mem_diff is W d_total_half[Q:] of rank 0 of a world-W external-collectives context on [x; y], within 1e-5."""
    Q, D = 96, 64
    m = (W - 1) * Q
    x, l, y, ly = _data(Q, m, D, 41 + W)
    xt, lt, yt, lyt = _dev(torch, x, l, y, ly)
    xall, lall = torch.cat([xt, yt]).contiguous(), torch.cat([lt, lyt]).contiguous()
    mem = _ctx(Q, D, m, FP16X2, USAGE)
    ext = capi.Context(capi.make_config(Q, D, world=W, rank=0, bwd_exchange=1, **USAGE))
    try:
        dx, dm = _mem_step(torch, mem, xt, lt, yt, lyt, 1.3)
        ext.forward_gathered(xall, lall)
        lh = torch.full((Q, D), float("nan"), device="cuda")
        th = torch.full((Q + m, D), float("nan"), device="cuda")
        ext.backward_partial(1.3, lh, th)
        torch.cuda.synchronize()
        ref = (W * th[Q:]).cpu().numpy()
        assert np.linalg.norm(dm - ref) <= 1e-5 * np.linalg.norm(ref)
        ref_x = (lh + W * th[:Q]).cpu().numpy()
        assert np.linalg.norm(dx - ref_x) <= 1e-5 * np.linalg.norm(ref_x)
    finally:
        mem.close(); ext.close()


# ---------------------------------------------------------------------------------------------------------- 5. refusals
def test_refusals_launch_nothing(torch):
    Q, D, M = 64, 32, 96
    x, l, y, ly = _data(Q, M, D, 43)
    xt, lt, yt, lyt = _dev(torch, x, l, y, ly)
    dx, dm = torch.empty_like(xt), torch.empty(M, D, device="cuda")
    lw = torch.ones(1, device="cuda")
    L = capi.lib()
    st = torch.cuda.current_stream().cuda_stream
    ctx = _ctx(Q, D, M)
    ring = capi.Context(capi.make_config(Q, D), memory_rows=M, ring=True)
    nofused = _ctx(Q, D, M, flags=capi.FLAG_NO_FUSED_GRAD)
    try:
        ctx.forward_memory(xt, lt, yt, lyt, M)
        ring.forward_ring(xt, lt)
        ring.forward_ring(xt, lt)
        nofused.forward_memory(xt, lt, yt, lyt, M)
        torch.cuda.synchronize()
        n0 = capi.kernel_launches()
        cases = [(ctx, dx.data_ptr(), None, -1), (ctx, None, dm.data_ptr(), -1), (ctx, dx.data_ptr() + 4, dm.data_ptr(), -1),
                 (ctx, dx.data_ptr(), dm.data_ptr() + 8, -1), (ring, dx.data_ptr(), dm.data_ptr(), -6),
                 (nofused, dx.data_ptr(), dm.data_ptr(), -1)]
        for c, a, b, code in cases:
            assert L.npair_backward_memory(c._h, C.c_float(1.0), a, b, st) == code, (a, b, code)
            assert L.npair_backward_memory_device_weight(c._h, lw.data_ptr(), a, b, st) == code, (a, b, code)
        assert L.npair_backward_memory_device_weight(ctx._h, None, dx.data_ptr(), dm.data_ptr(), st) == -1
        assert capi.kernel_launches() == n0
        ctx.forward(xt, lt)                                  # a forward that is not a memory forward
        torch.cuda.synchronize()
        n1 = capi.kernel_launches()
        assert L.npair_backward_memory(ctx._h, C.c_float(1.0), dx.data_ptr(), dm.data_ptr(), st) == -6
        assert L.npair_backward_memory_device_weight(ctx._h, lw.data_ptr(), dx.data_ptr(), dm.data_ptr(), st) == -6
        assert capi.kernel_launches() == n1
        fresh = _ctx(Q, D, M)
        try:
            n2 = capi.kernel_launches()
            assert L.npair_backward_memory(fresh._h, C.c_float(1.0), dx.data_ptr(), dm.data_ptr(), st) == -6   # no forward yet
            assert capi.kernel_launches() == n2
        finally:
            fresh.close()
        ctx.forward_memory(xt, lt, yt, lyt, M)               # the context is still usable
        ctx.backward_memory(1.0, dx, dm)
        torch.cuda.synchronize()
        assert torch.isfinite(dm).all()
    finally:
        ctx.close(); ring.close(); nofused.close()


# ---------------------------------------------------------------------------------------------------------- 6. capture
def test_captured_step_replays_the_eager_bits(torch):
    Q, D, m = 384, 96, 261
    batches = [_data(Q, m, D, 50 + b) for b in range(3)]
    ref = _ctx(Q, D, m, FP16X2, USAGE)
    ctx = _ctx(Q, D, m, FP16X2, USAGE)
    x, l, y, ly = (t.clone() for t in _dev(torch, *batches[0]))
    tops, lw = torch.zeros(5, device="cuda"), torch.ones(1, device="cuda")
    dx, dm = torch.zeros_like(x), torch.zeros_like(y)
    try:
        def enqueue():
            ctx.forward_memory_async(x, l, y, ly, m, tops)
            ctx.backward_memory_device_weight(lw, dx, dm)
        enqueue()                                            # warm-up: loads the kernels before the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            enqueue()
        for b, lwv in zip(range(3), (1.0, 0.5, 2.0)):
            for dst, src in zip((x, l, y, ly), _dev(torch, *batches[b])):
                dst.copy_(src)
            lw.fill_(lwv)
            g.replay()
            torch.cuda.synchronize()
            got = (dx.cpu().numpy(), dm.cpu().numpy())
            want = _mem_step(torch, ref, *_dev(torch, *batches[b]), lwv)
            for u, v, tag in zip(got, want, ("anchors", "memory rows")):
                np.testing.assert_array_equal(_bits(u), _bits(v), err_msg=f"replay {b} {tag}")
        ctx.async_status()
    finally:
        ctx.close(); ref.close()


# ---------------------------------------------------------------------------------------------------------- 7. torch
def test_proxy_gradient_matches_finite_differences(torch):
    """RAND mining (no thresholds: the loss is smooth): the proxies' gradient under true_gradient=True against central differences of
    the loss along random directions."""
    from npairloss_b200.torch_api import NPairLoss
    Q, D, C_ = 24, 16, 10
    x, l, _, _ = _data(Q, 0, D, 61, noise=1.5)
    rng = np.random.default_rng(5)
    p = rng.standard_normal((C_, D)).astype(np.float32)
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    xt, lt, pt = _dev(torch, x, l, p)
    lp = torch.arange(C_, device="cuda")
    fn = NPairLoss(true_gradient=True, sim_precision=BF16X3, **synth.DEFAULT_MINING)
    prox = pt.clone().requires_grad_(True)
    loss, _ = fn(xt, lt, extra_rows=prox, extra_labels=lp)
    loss.backward()
    g = prox.grad.double().cpu().numpy()
    assert np.abs(g).max() > 0
    for _ in range(4):
        v = rng.standard_normal((C_, D)).astype(np.float32)
        v /= np.linalg.norm(v)
        eps = 2e-2
        with torch.no_grad():
            up = float(fn(xt, lt, extra_rows=pt + eps * torch.from_numpy(v).cuda(), extra_labels=lp)[0])
            dn = float(fn(xt, lt, extra_rows=pt - eps * torch.from_numpy(v).cuda(), extra_labels=lp)[0])
        fd, an = (up - dn) / (2 * eps), float((g * v).sum())
        assert abs(fd - an) <= 2e-2 * abs(an) + 2e-4, (fd, an)


def _proxy_step(torch, fn, proxies, opt, x, l, lp):
    import torch.nn.functional as F
    opt.zero_grad(set_to_none=True)
    loss, _ = fn(x, l, extra_rows=F.normalize(proxies, dim=1), extra_labels=lp)
    loss.backward()
    opt.step()
    return loss


def test_proxy_training_step_captured_equals_eager(torch):
    """nn.Parameter proxies, NPairLoss(blocking=False) and SGD captured with torch.cuda.graph: four replays give, bit for bit, the
    loss and the proxies of eager blocking=True steps."""
    Q, D, C_ = 256, 128, 64
    data = [_dev(torch, *synth.make_inputs(Q, D, seed=70 + b, imgs_per_class=4, noise=1.0)) for b in range(6)]
    lp = torch.arange(C_, device="cuda").float()
    torch.manual_seed(7)
    init = torch.randn(C_, D, device="cuda")
    prox, prox_ref = torch.nn.Parameter(init.clone()), torch.nn.Parameter(init.clone())
    fn, fn_ref = (synth_loss(torch, blocking=False), synth_loss(torch, blocking=True))
    opt, opt_ref = torch.optim.SGD([prox], lr=0.5), torch.optim.SGD([prox_ref], lr=0.5)
    sx, sl = data[0][0].clone(), (data[0][1] % C_).clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for b in range(2):
            sx.copy_(data[b][0]); sl.copy_(data[b][1] % C_)
            _proxy_step(torch, fn, prox, opt, sx, sl, lp)
    torch.cuda.current_stream().wait_stream(side)
    for b in range(2):
        _proxy_step(torch, fn_ref, prox_ref, opt_ref, data[b][0], data[b][1] % C_, lp)
    g = torch.cuda.CUDAGraph()
    opt.zero_grad(set_to_none=True)
    with torch.cuda.graph(g):
        sloss = _proxy_step(torch, fn, prox, opt, sx, sl, lp)
    for b in range(2, 6):
        sx.copy_(data[b][0]); sl.copy_(data[b][1] % C_)
        g.replay()
        lr = _proxy_step(torch, fn_ref, prox_ref, opt_ref, data[b][0], data[b][1] % C_, lp)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(_bits(sloss), _bits(lr), err_msg=f"loss of batch {b}")
        np.testing.assert_array_equal(_bits(prox), _bits(prox_ref), err_msg=f"proxies after batch {b}")
    fn.async_status()


def synth_loss(torch, blocking):
    from npairloss_b200.torch_api import NPairLoss
    return NPairLoss(blocking=blocking, true_gradient=True, **USAGE)


def test_proxy_only_training_lowers_the_loss(torch):
    """Fixed clustered embeddings (classes of two rows), one learnable unit proxy per class: 40 SGD steps on the proxies alone lower
    the loss."""
    import torch.nn.functional as F
    from npairloss_b200.torch_api import NPairLoss
    Q, D, C_ = 256, 64, 128
    x, l = synth.make_inputs(Q, D, seed=80, imgs_per_class=2, noise=0.7)
    xt, lt = _dev(torch, x, l)
    classes = torch.unique(lt)
    assert classes.numel() == C_
    torch.manual_seed(3)
    prox = torch.nn.Parameter(F.normalize(torch.randn(C_, D, device="cuda"), dim=1))
    fn = NPairLoss(true_gradient=True, **synth.DEFAULT_MINING)
    opt = torch.optim.SGD([prox], lr=20.0)
    losses = []
    for _ in range(40):
        opt.zero_grad(set_to_none=True)
        loss, _ = fn(xt, lt, extra_rows=F.normalize(prox, dim=1), extra_labels=classes)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    print(f"proxy-only training: loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert losses[-1] < losses[0] - 0.01, losses
