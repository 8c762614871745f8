"""Per-anchor loss weights and per-anchor losses (npair_set_anchor_io, DESIGN 4.5) on the GPU.

- No weights and w = 1 give the unweighted forward and backward bit for bit on every path: tops, gradient, every npair_debug_read
  array and the row records.
- The weighted loss and gradient match the weighted oracle run on the GPU's own S (thresholds bit for bit, loss 1e-5, gradient 1e-5
  normwise), and the gradient matches fp64 under the rules of test_gpu_grad_precision.
- The weighted records are the unweighted ones with m2c - log2f(w), cA w, cT w; row_loss is -log(A/T) bit for bit.
- Masking, invalid weights, and the torch API (finite differences, the weights' gradient, graph capture)."""
import itertools

import numpy as np
import pytest

import forward_ref
import grad_ref
from grad_ref import SGEMM_FACTOR
from npairloss_b200 import capi, synth, torch_api
from oracle import npair_oracle_np as onp

pytestmark = pytest.mark.gpu

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
TC, SIMT = capi.GEMM_TCGEN05, capi.GEMM_SIMT_CHECK
E_ARG = -1
USAGE = dict(synth.USAGE_MINING)
RAND = dict(synth.DEFAULT_MINING)
LOCAL_SN = dict(ap_region=capi.LOCAL, ap_method=capi.RELATIVE_HARD, an_region=capi.LOCAL, an_method=capi.RELATIVE_HARD, identsn=-0.4,
                diffsn=-0.3, margin_diff=-0.02)
DEBUG_ARRAYS = (1, 2, 3, 4, 5, 6, 7, 8, 9, 11, 12)


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _cuda(torch, *arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _state(torch, ctx, Q):
    """Every per-row array the forward leaves (npair_debug_read), the row records and, when there is one, nothing else."""
    st = {k: ctx.debug_read(k, 3 * Q if k == 12 else Q) for k in DEBUG_ARRAYS}
    rec = torch.empty(Q * 8, dtype=torch.float32, device="cuda")
    ctx.row_scalars(rec)
    torch.cuda.synchronize()
    st["rec"] = rec.cpu().numpy().reshape(Q, 8)
    return st


def _step(torch, ctx, x, l, w=None, rl=None, set_io=True, mem=None, lw=0.75, mode="sync"):
    """One forward + backward through ctx, anchor IO set before (set_io) and cleared after: (tops, dx, state)."""
    Q = x.shape[0]
    if set_io:
        ctx.set_anchor_io(w, rl)
    dx = torch.full_like(x, float("nan"))
    if mode == "sync":
        tops = np.array(ctx.forward(x, l) if mem is None else ctx.forward_memory(x, l, *mem), np.float32)
        ctx.backward(lw, dx)
    else:
        t = torch.full((5,), 7.0, device="cuda")
        if mem is None:
            ctx.forward_async(x, l, t)
        else:
            ctx.forward_memory_async(x, l, *mem, t)
        ctx.backward_device_weight(torch.tensor([lw], dtype=torch.float32, device="cuda"), dx)
        torch.cuda.synchronize()
        tops = t.cpu().numpy()
    if set_io:
        ctx.set_anchor_io(None, None)
    torch.cuda.synchronize()
    return tops, dx.cpu().numpy(), _state(torch, ctx, Q)


def _same_bits(a, b, tag):
    ta, da, sa = a
    tb, db, sb = b
    np.testing.assert_array_equal(_bits(ta), _bits(tb), err_msg=f"{tag} tops")
    np.testing.assert_array_equal(_bits(da), _bits(db), err_msg=f"{tag} gradient")
    for k in sa:
        np.testing.assert_array_equal(_bits(sa[k]), _bits(sb[k]), err_msg=f"{tag} debug array {k}")


# ------------------------------------------------------------------------------------------------ bit for bit: none / w = 1
WORLD1_PATHS = {
    "fp16x2 fused": dict(sim_precision=FP16X2),
    "fp16x2 split": dict(sim_precision=FP16X2, flags=capi.FLAG_NO_FUSED_GRAD),
    "bf16x3 fused": dict(sim_precision=BF16X3),
    "bf16x3 split": dict(sim_precision=BF16X3, flags=capi.FLAG_NO_FUSED_GRAD),
    "bf16 fused": dict(sim_precision=BF16),
    "simt": dict(gemm_backend=SIMT),
    "row blocks": dict(sim_block_rows=128),
    "global_scope": dict(global_scope=1),
    "normalize_input": dict(normalize_input=1),
}


@pytest.mark.parametrize("mining", ["usage", "local_sn"])
@pytest.mark.parametrize("path", list(WORLD1_PATHS))
def test_unit_weights_bit_for_bit(torch, path, mining):
    """No npair_set_anchor_io, NULL pointers, and w = 1 with a row-loss output: the same bits everywhere; row_loss = -logv."""
    Q, D = 333, 72
    x, l = _cuda(torch, *synth.make_inputs(Q, D, seed=41, imgs_per_class=3, noise=1.5))
    ctx = capi.Context(capi.make_config(Q, D, **(USAGE if mining == "usage" else LOCAL_SN), **WORLD1_PATHS[path]))
    try:
        ref = _step(torch, ctx, x, l, set_io=False)
        _same_bits(ref, _step(torch, ctx, x, l, None, None), f"{path} NULL")
        rl = torch.full((Q,), 5.0, device="cuda")
        _same_bits(ref, _step(torch, ctx, x, l, torch.ones(Q, device="cuda"), rl), f"{path} w = 1")
        np.testing.assert_array_equal(_bits(rl.cpu().numpy()), _bits(-ref[2][11]), err_msg=f"{path} row_loss")
        rl.fill_(5.0)
        _same_bits(ref, _step(torch, ctx, x, l, None, rl), f"{path} row_loss only")
        np.testing.assert_array_equal(_bits(rl.cpu().numpy()), _bits(-ref[2][11]), err_msg=f"{path} row_loss only")
    finally:
        ctx.close()


@pytest.mark.parametrize("m", [0, 200])
@pytest.mark.parametrize("mode", ["sync", "async"])
def test_unit_weights_bit_for_bit_memory_and_async(torch, m, mode):
    Q, D = 256, 64
    x, lab = synth.make_inputs(Q + max(m, 1), D, seed=43, imgs_per_class=2, noise=1.5)
    xt, lt, xm, lm = _cuda(torch, x[:Q], lab[:Q], x[Q:Q + m] if m else x[Q:Q + 1], lab[Q:Q + m] if m else lab[Q:Q + 1])
    ctx = capi.Context(capi.make_config(Q, D, **USAGE), memory_rows=256)
    try:
        mem = (xm, lm, m)
        ref = _step(torch, ctx, xt, lt, set_io=False, mem=mem, mode=mode)
        _same_bits(ref, _step(torch, ctx, xt, lt, torch.ones(Q, device="cuda"), None, mem=mem, mode=mode), f"memory {m} {mode}")
        if mode == "async":
            ctx.async_status()
    finally:
        ctx.close()


def test_unit_weights_bit_for_bit_graph_replay(torch):
    """A captured step with w = 1 replays the eager unweighted step's bits; new weights copied into the static tensor take effect."""
    Q, D = 512, 64
    x, l = _cuda(torch, *synth.make_inputs(Q, D, seed=44, imgs_per_class=4, noise=1.5))
    w = torch.ones(Q, device="cuda")
    rl = torch.zeros(Q, device="cuda")
    ctx = capi.Context(capi.make_config(Q, D, **USAGE))
    try:
        ref = _step(torch, ctx, x, l, set_io=False)
        w2 = torch.from_numpy(grad_ref.make_weights(Q, np.random.default_rng(4))).cuda()
        ref2 = _step(torch, ctx, x, l, w2, None)
        tops = torch.zeros(5, device="cuda")
        dx = torch.zeros_like(x)
        lw = torch.tensor([0.75], device="cuda")
        s = torch.cuda.Stream()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            ctx.set_anchor_io(w, rl)
            with torch.cuda.graph(g, stream=s):
                ctx.forward_async(x, l, tops)
                ctx.backward_device_weight(lw, dx)
            ctx.set_anchor_io(None, None)
        for weights, r, tag in ((None, ref, "w = 1"), (w2, ref2, "new weights")):
            if weights is not None:
                w.copy_(weights)
            g.replay()
            torch.cuda.synchronize()
            np.testing.assert_array_equal(_bits(tops.cpu().numpy()), _bits(r[0]), err_msg=f"replay {tag} tops")
            np.testing.assert_array_equal(_bits(dx.cpu().numpy()), _bits(r[1]), err_msg=f"replay {tag} gradient")
            np.testing.assert_array_equal(_bits(rl.cpu().numpy()), _bits(-r[2][11]), err_msg=f"replay {tag} row_loss")
        ctx.async_status()
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ emulated ranks
def _world_step(torch, x, lab, Q, world, w, mining, bwd_exchange, prec=FP16X2, lw=0.7):
    """gpu_harness.gpu_step_world with each rank's Q weights set (w None: no npair_set_anchor_io); also the ranks' records and
    row losses."""
    N, D = x.shape
    xt, lt = _cuda(torch, x, lab)
    tops = np.zeros((world, 5), np.float32)
    S = np.zeros((N, N), np.float32)
    local = torch.zeros((N, D), device="cuda")
    total = torch.zeros((N, D), device="cuda")
    wt = None if w is None else torch.from_numpy(np.ascontiguousarray(w, dtype=np.float32)).cuda()
    rl = torch.full((N,), 9.0, device="cuda")
    rs = torch.empty((world, Q, 8), device="cuda")
    ctxs = []
    try:
        for r in range(world):
            ctx = capi.Context(capi.make_config(Q, D, world=world, rank=r, sim_precision=prec, bwd_exchange=bwd_exchange, **mining))
            ctxs.append(ctx)
            if wt is not None:
                ctx.set_anchor_io(wt[r * Q:(r + 1) * Q], rl[r * Q:(r + 1) * Q])
            tops[r] = ctx.forward_gathered(xt, lt)
            S[r * Q:(r + 1) * Q] = ctx.debug_read(0, Q * N).reshape(Q, N)
            ctx.row_scalars(rs[r])
        mode = ctxs[0].bwd_exchange_mode()
        for r in range(world):
            if mode == 2:
                g = torch.full((Q, D), float("nan"), device="cuda")
                ctxs[r].backward_gathered(lw, rs, g)
                local[r * Q:(r + 1) * Q] = g
            else:
                lh = torch.full((Q, D), float("nan"), device="cuda")
                th = torch.full((N, D), float("nan"), device="cuda")
                ctxs[r].backward_partial(lw, lh, th)
                local[r * Q:(r + 1) * Q] = lh
                total += th
        logv = np.concatenate([c.debug_read(11, Q) for c in ctxs])
    finally:
        for c in ctxs:
            c.close()
    torch.cuda.synchronize()
    return dict(tops=tops, dx=(local + total).cpu().numpy(), S=S, rec=rs.cpu().numpy().reshape(N, 8), rl=rl.cpu().numpy(), logv=logv,
                mode=mode)


@pytest.mark.parametrize("bwd_exchange", [0, 1], ids=["records", "reduce_scatter"])
@pytest.mark.parametrize("world", [2, 3])
def test_emulated_world(torch, oracle, world, bwd_exchange):
    """Both exchange forms: w = 1 is the unweighted step bit for bit; random weights match the weighted oracle on the GPU's S, and the
    records carry them."""
    Q, D = 160, 48
    x, lab = synth.make_inputs(Q * world, D, seed=50 + world, imgs_per_class=3, noise=1.0)
    N = Q * world
    for mining in (USAGE, LOCAL_SN):
        ref = _world_step(torch, x, lab, Q, world, None, mining, bwd_exchange)
        one = _world_step(torch, x, lab, Q, world, np.ones(N, np.float32), mining, bwd_exchange)
        for k in ("tops", "dx", "S", "rec"):
            np.testing.assert_array_equal(_bits(one[k]), _bits(ref[k]), err_msg=f"w{world} x{bwd_exchange} w = 1 {k}")
        np.testing.assert_array_equal(_bits(one["rl"]), _bits(-ref["logv"]))
        w = grad_ref.make_weights(N, np.random.default_rng(world))
        g = _world_step(torch, x, lab, Q, world, w, mining, bwd_exchange)
        np.testing.assert_array_equal(_bits(g["S"]), _bits(ref["S"]))
        _check_records(g["rec"], ref["rec"], w, f"w{world} x{bwd_exchange}")
        cfg = oracle.make_config(Q, D, world=world, faithful_sorts=0, **mining)
        tops_o, dx_o = oracle.step_world(x, lab, cfg, 0.7, S_inject_all=g["S"], anchor_weight=w)
        _check_oracle(g["tops"], g["dx"], tops_o, dx_o, f"w{world} x{bwd_exchange}")
        np.testing.assert_array_equal(g["tops"][:, 1:], ref["tops"][:, 1:])


def _check_records(rec_w, rec_1, w, tag):
    """Records bit for bit the weighted model of the unweighted ones, m2c within an ulp of log2 where w is no power of two."""
    model = forward_ref.weighted_records(rec_1, w)
    keep = [1, 2, 3, 4, 5, 6, 7]
    np.testing.assert_array_equal(_bits(rec_w[:, keep]), _bits(model[:, keep]), err_msg=f"{tag} records")
    dyadic = (w == 0) | (np.frexp(w)[0] == 0.5)
    np.testing.assert_array_equal(_bits(rec_w[dyadic, 0]), _bits(model[dyadic, 0]), err_msg=f"{tag} m2c at w = 0, 2^-j")
    m1, mw = rec_w[~dyadic, 0], model[~dyadic, 0]
    fin = np.isfinite(mw)
    assert np.array_equal(np.isfinite(m1), fin), tag
    lg = np.abs(np.log2(w[~dyadic]).astype(np.float32))
    assert np.all(np.abs(m1[fin] - mw[fin]) <= np.spacing(np.abs(mw[fin])) + np.spacing(lg[fin])), f"{tag} m2c"


def _check_oracle(tops, dx, tops_o, dx_o, tag, g_tol=1e-5):
    np.testing.assert_allclose(tops[:, 0], tops_o[:, 0], rtol=1e-5, atol=1e-6, err_msg=f"{tag} loss")
    assert np.isfinite(dx).all(), f"{tag} non-finite gradient"
    gn = float(np.linalg.norm(dx_o))
    assert float(np.linalg.norm(dx - dx_o)) <= g_tol * max(gn, 1e-20), f"{tag} gradient {np.linalg.norm(dx - dx_o) / max(gn, 1e-20):.2e}"


# ------------------------------------------------------------------------------------------------ weighted oracle parity (L2)
@pytest.mark.parametrize("backend", [TC, SIMT])
def test_all_mining_modes_weighted(torch, oracle, backend):
    """Every (region, method) combination, weights with zeros, the weighted oracle on the GPU's own S; thresholds bit for bit."""
    Q, D = 48, 40
    x, lab = synth.make_inputs(Q, D, seed=101, imgs_per_class=3, noise=0.7)
    w = grad_ref.make_weights(Q, np.random.default_rng(60))
    xt, lt, wt = _cuda(torch, x, lab, w)
    for apR, apM, anR, anM in itertools.product([0, 1], range(5), [0, 1], range(5)):
        mining = dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3, ap_region=apR, ap_method=apM, an_region=anR,
                      an_method=anM)
        tag = f"b{backend} {apR}{apM}{anR}{anM}"
        ctx = capi.Context(capi.make_config(Q, D, gemm_backend=backend, **mining))
        try:
            ctx.set_anchor_io(wt, None)
            tops = np.array(ctx.forward(xt, lt), np.float32)[None]
            dx = torch.full_like(xt, float("nan"))
            ctx.backward(0.7, dx)
            torch.cuda.synchronize()
            S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
            posi, nega = ctx.debug_read(1, Q), ctx.debug_read(2, Q)
        finally:
            ctx.close()
        _, st = oracle.forward(x, lab, oracle.make_config(Q, D, faithful_sorts=0, **mining), S_inject=S)
        np.testing.assert_array_equal(posi, st["posi_thr"], err_msg=tag)
        np.testing.assert_array_equal(nega, st["nega_thr"], err_msg=tag)
        cfg = oracle.make_config(Q, D, faithful_sorts=0, **mining)
        tops_o, dx_o = oracle.step_world(x, lab, cfg, 0.7, S_inject_all=S, anchor_weight=w)
        _check_oracle(tops, dx.cpu().numpy(), tops_o, dx_o, tag)


@pytest.mark.parametrize("prec", [FP16X2, BF16X3])
@pytest.mark.parametrize("Q,D", [(5, 3), (129, 33), (257, 130), (999, 101)])
def test_ragged_shapes_weighted(torch, oracle, Q, D, prec):
    x, lab = synth.make_inputs(Q, D, seed=Q + D, imgs_per_class=3, noise=1.0)
    w = grad_ref.make_weights(Q, np.random.default_rng(Q))
    xt, lt, wt = _cuda(torch, x, lab, w)
    rl = torch.zeros(Q, device="cuda")
    ctx = capi.Context(capi.make_config(Q, D, sim_precision=prec, **RAND))
    try:
        ref = _step(torch, ctx, xt, lt, set_io=False)
        tw, dxw, stw = _step(torch, ctx, xt, lt, wt, rl)
        S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
    finally:
        ctx.close()
    tag = f"Q {Q} D {D}"
    _check_records(stw["rec"], ref[2]["rec"], w, tag)
    np.testing.assert_array_equal(_bits(rl.cpu().numpy()), _bits(-ref[2][11]), err_msg=tag)
    for k in DEBUG_ARRAYS:
        np.testing.assert_array_equal(_bits(stw[k]), _bits(ref[2][k]), err_msg=f"{tag} debug array {k}")
    np.testing.assert_array_equal(tw[1:], ref[0][1:])
    cfg = oracle.make_config(Q, D, faithful_sorts=0, **RAND)
    tops_o, dx_o = oracle.step_world(x, lab, cfg, 0.75, S_inject_all=S, anchor_weight=w)
    _check_oracle(tw[None], dxw, tops_o, dx_o, tag)


# ------------------------------------------------------------------------------------------------ against fp64
def _check_fp64(dx, ref, prec, path, N, tag, clustered):
    k = SGEMM_FACTOR["accumulator" if clustered or path == "split" else "spread"]
    rel = max(1e-5, 2e-4) if path == "split" else 1e-5
    bad, m = grad_ref.violations(dx, ref, grad_ref.tau(prec, path, N), rel=rel, k_sgemm=k)
    print(f"{tag} {path}: normwise {m['normwise']:.2e} worst row {m['row']:.3f} componentwise {m['comp']:.1f} x 2^-24 of B")
    assert not bad, f"{tag} {path}: " + "; ".join(bad)


@pytest.mark.parametrize("path", ["fused", "split"])
@pytest.mark.parametrize("kind,Q,D", [("synth", 1000, 200), ("0.02", 1000, 200), ("synth", 8192, 512), ("0.02", 8192, 512)])
def test_gradient_against_fp64(torch, kind, Q, D, path):
    """Weighted gradient against fp64 (grad_ref's rules) on spread and clustered rows, up to the flagship shape."""
    x, lab = synth.make_inputs(Q, D, 12, noise=2.5) if kind == "synth" else grad_ref.cone_inputs(Q, D, float(kind), 12)
    w = grad_ref.make_weights(Q, np.random.default_rng(Q))
    xt, lt, wt = _cuda(torch, x, lab, w)
    flags = capi.FLAG_NO_FUSED_GRAD if path == "split" else 0
    ctx = capi.Context(capi.make_config(Q, D, num_tops=2, flags=flags, **RAND))
    try:
        ctx.set_anchor_io(wt, None)
        ctx.forward(xt, lt)
        dx = torch.full_like(xt, float("nan"))
        ctx.backward(1.0, dx)
        torch.cuda.synchronize()
        S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
    finally:
        ctx.close()
    ref = grad_ref.step(x, lab, Q, 1, S, w, **RAND)
    _check_fp64(dx.cpu().numpy(), ref, FP16X2, path, Q, f"{kind} {Q}", kind != "synth")


@pytest.mark.parametrize("Q,m", [(1024, 7168)])
def test_memory_step_against_fp64(torch, Q, m):
    D = 128
    x, lab = grad_ref.cone_inputs(Q + m, D, 0.1, 19)
    lab = np.concatenate([lab[:Q], lab[Q:] % (Q // 2)]).astype(np.float32)
    w = grad_ref.make_weights(Q, np.random.default_rng(m))
    xt, lt, xm, lm, wt = _cuda(torch, x[:Q], lab[:Q], x[Q:], lab[Q:], w)
    ctx = capi.Context(capi.make_config(Q, D, num_tops=2, **USAGE), memory_rows=m)
    try:
        ctx.set_anchor_io(wt, None)
        ctx.forward_memory(xt, lt, xm, lm, m)
        dx = torch.full_like(xt, float("nan"))
        ctx.backward(1.0, dx)
        torch.cuda.synchronize()
        S = ctx.debug_read(0, Q * (Q + m)).reshape(Q, Q + m)
    finally:
        ctx.close()
    ref = grad_ref.step(x, lab, Q, 1, S, w, **USAGE)
    ref = {k: ref[k][:Q] for k in ("R", "B", "R32")}                            # the anchors' rows
    _check_fp64(dx.cpu().numpy(), ref, FP16X2, "fused", Q + m, f"memory Q {Q} m {m}", True)


# ------------------------------------------------------------------------------------------------ masking and invalid weights
def test_masking_and_all_zero(torch, oracle):
    """A row with w = 0 keeps the gradient it gets as the other anchors' column (the oracle's G with row i zeroed); every w = 0 gives
    loss 0, an all-zero gradient, and the unweighted tops 1-4."""
    Q, D = 200, 32
    x, lab = synth.make_inputs(Q, D, seed=70, imgs_per_class=4, noise=1.0)
    xt, lt = _cuda(torch, x, lab)
    w = np.ones(Q, np.float32)
    w[::3] = 0.0
    ctx = capi.Context(capi.make_config(Q, D, **USAGE))
    try:
        ref = _step(torch, ctx, xt, lt, set_io=False)
        S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
        t, dx, _ = _step(torch, ctx, xt, lt, *_cuda(torch, w), None)
        tz, dxz, _ = _step(torch, ctx, xt, lt, torch.zeros(Q, device="cuda"), None)
    finally:
        ctx.close()
    cfg = oracle.make_config(Q, D, faithful_sorts=0, **USAGE)
    tops_o, dx_o = oracle.step_world(x, lab, cfg, 0.75, S_inject_all=S, anchor_weight=w)
    _check_oracle(t[None], dx, tops_o, dx_o, "masked")
    _, only_cols = onp.step_world(x, lab, Q, 1, 0.75, S_inject_all=S, anchor_weight=w, **USAGE)
    masked = w == 0
    assert np.linalg.norm(dx[masked] - only_cols[masked]) <= 1e-5 * np.linalg.norm(only_cols[masked])
    assert tz[0] == 0.0 and np.all(dxz == 0.0)
    np.testing.assert_array_equal(tz[1:], ref[0][1:])


@pytest.mark.parametrize("bad", [-0.5, 1.5, float("nan")])
def test_invalid_weights(torch, bad):
    Q, D = 64, 16
    xt, lt = _cuda(torch, *synth.make_inputs(Q, D, seed=71, imgs_per_class=2))
    w = torch.ones(Q, device="cuda")
    w[17] = bad
    ctx = capi.Context(capi.make_config(Q, D, **USAGE))
    try:
        ref = np.array(ctx.forward(xt, lt), np.float32)
        ctx.set_anchor_io(w, None)
        with pytest.raises(capi.NpairError) as e:
            ctx.forward(xt, lt)
        assert e.value.code == E_ARG and "anchor weight" in str(e.value)
        tops = torch.zeros(5, device="cuda")
        ctx.forward_async(xt, lt, tops)
        torch.cuda.synchronize()
        assert np.all(np.isnan(tops.cpu().numpy()))
        with pytest.raises(capi.NpairError) as e:
            ctx.async_status()
        assert e.value.code == E_ARG
        ctx.async_status()                              # cleared
        w[17] = 1.0
        np.testing.assert_array_equal(np.array(ctx.forward(xt, lt), np.float32), ref)
        ctx.set_anchor_io(None, None)
        np.testing.assert_array_equal(np.array(ctx.forward(xt, lt), np.float32), ref)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ torch
def test_torch_finite_differences_and_weight_gradient(torch):
    """true_gradient: directional finite differences of the weighted loss (fp64 steps of an fp32 loss, bf16x3 operands, every pair
    selected); the weights' gradient is row_loss / Q."""
    Q, D = 32, 16
    x, lab = synth.make_inputs(Q, D, seed=72, imgs_per_class=4, noise=1.0)
    w = grad_ref.make_weights(Q, np.random.default_rng(72))
    m = torch_api.NPairLoss(true_gradient=True, sim_precision=BF16X3, **RAND)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    wt = torch.from_numpy(w).cuda().requires_grad_(True)
    lt = torch.from_numpy(lab).cuda()
    loss, tops, rl = m(xt, lt, anchor_weight=wt, row_losses=True)
    loss.backward()
    g = xt.grad.double().cpu().numpy()
    np.testing.assert_allclose(wt.grad.cpu().numpy(), rl.cpu().numpy() / Q, rtol=1e-6)
    assert float(loss.detach()) == pytest.approx(float((wt.detach() * rl).sum()) / Q, rel=1e-5)
    rng = np.random.default_rng(0)
    h = 1e-2
    for _ in range(4):
        v = rng.standard_normal(x.shape).astype(np.float32)
        v /= np.linalg.norm(v)
        vt = torch.from_numpy(v).cuda()
        with torch.no_grad():
            lp = float(m(xt.detach() + h * vt, lt, anchor_weight=wt.detach())[0])
            lm = float(m(xt.detach() - h * vt, lt, anchor_weight=wt.detach())[0])
        fd = (lp - lm) / (2 * h)
        assert fd == pytest.approx(float((g * v).sum()), rel=2e-2, abs=2e-5)


def test_torch_graph_step_with_weights(torch):
    """A whole step with weights under torch.cuda.graph, replayed with new weights copied into the static tensor: bit for bit the
    eager blocking=True step."""
    Q, D = 256, 64
    x, lab = synth.make_inputs(Q, D, seed=73, imgs_per_class=4, noise=1.5)
    static_x = torch.from_numpy(x).cuda()
    static_l = torch.from_numpy(lab).cuda()
    static_w = torch.ones(Q, device="cuda")
    eager = torch_api.NPairLoss(**USAGE)
    graphed = torch_api.NPairLoss(blocking=False, **USAGE)
    xg = static_x.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                        # warm-up: the context and the autograd graph
        loss, tops, rl = graphed(xg, static_l, anchor_weight=static_w, row_losses=True)
        loss.backward()
    torch.cuda.current_stream().wait_stream(s)
    del loss, tops, rl                                # the warm-up's autograd graph
    xg.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        loss, tops, rl = graphed(xg, static_l, anchor_weight=static_w, row_losses=True)
        loss.backward()
    rng = np.random.default_rng(5)
    for _ in range(2):
        w = torch.from_numpy(grad_ref.make_weights(Q, rng)).cuda()
        static_w.copy_(w)
        g.replay()
        torch.cuda.synchronize()
        xe = static_x.clone().requires_grad_(True)
        le, te, rle = eager(xe, static_l, anchor_weight=w, row_losses=True)
        le.backward()
        torch.cuda.synchronize()
        np.testing.assert_array_equal(_bits(tops.cpu().numpy()), _bits(te.cpu().numpy()))
        np.testing.assert_array_equal(_bits(xg.grad.cpu().numpy()), _bits(xe.grad.cpu().numpy()))
        np.testing.assert_array_equal(_bits(rl.cpu().numpy()), _bits(rle.cpu().numpy()))
    graphed.async_status()
