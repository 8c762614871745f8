"""GPU parity at the shapes and buffers where the layer's kernels take their less travelled paths: D not a multiple of 8 (the
operand split's per-element loads, the gradient drains' scalar stores), Q next to the 128-row tile and symmetric-tile boundaries,
a ragged second 256-column gradient tile, split-K whose slices are not 16-byte aligned (Q*D % 4 != 0), rank offsets that are no
multiple of 8, the unfused cross-check gradient, non-default accumulation chunks, feature and label buffers at any offset, gradient
outputs that are not 16-byte aligned (refused), and batches of two or three rows."""
import numpy as np
import pytest

from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
PRECS = [FP16X2, BF16X3, BF16]
PREC_NAME = {BF16X3: "bf16x3", BF16: "bf16", FP16X2: "fp16x2"}
TC = capi.GEMM_TCGEN05

MININGS = {
    "usage": synth.USAGE_MINING,
    "local_rel": dict(synth.DEFAULT_MINING, ap_method=capi.RELATIVE_HARD, an_method=capi.RELATIVE_HARD, identsn=0.0, diffsn=-0.3,
                      margin_diff=-0.01),
    "global_hard": dict(synth.DEFAULT_MINING, ap_region=capi.GLOBAL, ap_method=capi.HARD, an_region=capi.GLOBAL, an_method=capi.HARD,
                        margin_diff=-0.05),
}
ORACLE_TO_NPAIR = {1: -1, 2: -4, 3: -5}       # NPO_ERR_* -> NPAIR_E_*


@pytest.fixture(scope="module")
def cuda():
    import torch
    assert torch.cuda.is_available(), "GPU tests need an H100"
    assert torch.cuda.get_device_capability(0) == (9, 0)
    return torch


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


def grad_splits(Q, D, world, prec, fused, sms):
    """split_k (host.cuh) restated: split-K slices of the rank's Q x D gradient GEMM, whose K is the N = Q*world sample index in blocks
    of 32 (fused kernel, >= 8 blocks per slice) or of the split GEMM's K block (>= 4 per slice), on 128 x 256 output tiles."""
    kb = _cdiv(Q * world, 32 if fused or prec != BF16 else 64)
    tiles = _cdiv(Q, 128) * _cdiv(D, 256)
    s = max(1, min(sms // tiles, 16, kb // (8 if fused else 4)))
    return _cdiv(kb, _cdiv(kb, s))


def _inputs(B, D, seed, noise=1.0):
    """Two images per class; an odd batch's last image joins the class before it, so every row has a positive."""
    x, lab = synth.make_inputs(B, D, seed, imgs_per_class=2, noise=noise)
    if B % 2:
        lab[-1] = lab[-2]
    return x, lab


# ---------------------------------------------------------------------------------------------------- ragged shapes
QS = (127, 129, 255, 257, 385)                  # around the 128-row tiles and the symmetric tile list's mb/2 boundary
DS = (1, 3, 33, 65, 101, 130, 257, 300)         # D % 8 != 0; 257 and 300: a ragged second 256-column gradient tile


def _grid():
    """Each mining meets every D and every Q (not the whole cross product): D k goes with Q (k + 2m) % 5 under mining m."""
    return [pytest.param(name, QS[(k + 2 * m) % len(QS)], D, id=f"{name}-Q{QS[(k + 2 * m) % len(QS)]}-D{D}")
            for m, name in enumerate(MININGS) for k, D in enumerate(DS)]


@pytest.mark.parametrize("mining_name,Q,D", _grid())
def test_ragged_shapes(cuda, oracle, mining_name, Q, D):
    """D = 1: S = +-1 everywhere, so every mining rule meets exact ties."""
    from gpu_harness import check_parity
    x, lab = _inputs(Q, D, seed=1000 * Q + D, noise=2.5)
    r = check_parity(oracle, x, lab, Q, 1, MININGS[mining_name], FP16X2, TC, loss_weight=0.7, tag=f"{mining_name} Q{Q} D{D}")
    print(mining_name, Q, D, r)


# ---------------------------------------------------------------------------------------------------- split-K
# Q*D % 4 = 3, 2, 1: slices 1.. of the split-K partial products start off the 16-byte grid
SPLITK_SHAPES = [(999, 101), (1001, 130), (513, 257)]


@pytest.mark.parametrize("prec", PRECS, ids=lambda p: PREC_NAME[p])
@pytest.mark.parametrize("Q,D", SPLITK_SHAPES)
def test_split_k_with_unaligned_slices(cuda, oracle, Q, D, prec):
    """The fused gradient kernel splits K and splitk_reduce_kernel sums slices that are not 16-byte aligned (its scalar path)."""
    from gpu_harness import check_parity
    splits = grad_splits(Q, D, 1, prec, True, _sms())
    assert splits > 1 and (Q * D) % 4, (splits, Q * D % 4)
    x, lab = _inputs(Q, D, seed=Q + D)
    r = check_parity(oracle, x, lab, Q, 1, synth.DEFAULT_MINING, prec, TC, loss_weight=0.7, tag=f"Q{Q} D{D} {PREC_NAME[prec]}")
    print(Q, D, PREC_NAME[prec], f"splits {splits}", r)


# ---------------------------------------------------------------------------------------------------- emulated ranks
@pytest.mark.parametrize("bwd_exchange", [0, 1])
@pytest.mark.parametrize("Q,world,D", [(333, 3, 101), (129, 2, 257)])
def test_emulated_ranks_at_ragged_sizes(cuda, oracle, Q, world, D, bwd_exchange):
    """Rank offsets 129, 333 and 666 are no multiple of 8 (split_tile's per-element stores of the local transposed operand in the
    reduce-scatter form); that form's local GEMM splits K over slices of Q*D % 4 = 1 floats."""
    from gpu_harness import check_parity
    x, lab = _inputs(Q * world, D, seed=Q * world + D, noise=2.5)
    fused = bwd_exchange == 0
    splits = grad_splits(Q, D, world, FP16X2, fused, _sms())
    if not fused or (Q, D) == (333, 101):
        assert splits > 1, splits
    r = check_parity(oracle, x, lab, Q, world, synth.USAGE_MINING, FP16X2, TC, loss_weight=0.7, bwd_exchange=bwd_exchange,
                     tag=f"Q{Q} w{world} D{D} x{bwd_exchange}")
    print(Q, world, D, bwd_exchange, f"splits {splits}", r)


# ---------------------------------------------------------------------------------------------------- cross-check path
@pytest.mark.parametrize("Q,D", [(999, 101), (1024, 128)])
def test_unfused_gradient_cross_check(cuda, oracle, Q, D):
    """NPAIR_FLAG_NO_FUSED_GRAD at world 1 on the tensor cores: the BW_SYM weight builder, then the split GEMM's EPI_OUT drain and
    the split-K reduce.  Both gradient paths meet the oracle, and each other within twice its tolerance (they accumulate in
    different orders, so they are not bitwise equal)."""
    from gpu_harness import G_TOL, check_parity, gpu_step_world
    x, lab = _inputs(Q, D, seed=Q * D)
    for flags in (capi.FLAG_NO_FUSED_GRAD, 0):
        assert grad_splits(Q, D, 1, FP16X2, flags == 0, _sms()) > 1
        check_parity(oracle, x, lab, Q, 1, synth.DEFAULT_MINING, FP16X2, TC, loss_weight=0.7, tag=f"Q{Q} D{D} flags {flags}", flags=flags)
    dx = [gpu_step_world(x, lab, Q, 1, synth.DEFAULT_MINING, FP16X2, TC, loss_weight=0.7, flags=f)["dx"] for f in (capi.FLAG_NO_FUSED_GRAD, 0)]
    rel = float(np.linalg.norm(dx[0] - dx[1]) / np.linalg.norm(dx[1]))
    print(Q, D, f"unfused vs fused gradient: normwise {rel:.3e}")
    assert rel <= 2 * G_TOL[FP16X2], rel


# ---------------------------------------------------------------------------------------------------- accumulation chunks
@pytest.mark.parametrize("chunk", [32, 96, 1024, 0, -1])
@pytest.mark.parametrize("Q,D", [(2048, 512), (999, 101)])
def test_grad_chunk_cols(cuda, oracle, Q, D, chunk):
    """grad_chunk_cols: one- and three-block chunks (the first chunk of a tile shortened to max(1, ...) blocks), 1024, the default
    and one accumulator per slice.  On 132 SMs, (2048, 512): 4 slices of 16 K blocks; (999, 101): 4 slices of 8."""
    from gpu_harness import check_parity
    assert grad_splits(Q, D, 1, FP16X2, True, _sms()) > 1
    x, lab = _inputs(Q, D, seed=Q + D + 7)
    r = check_parity(oracle, x, lab, Q, 1, synth.DEFAULT_MINING, FP16X2, TC, tag=f"Q{Q} D{D} chunk {chunk}", grad_chunk_cols=chunk)
    print(f"Q{Q} D{D} grad_chunk_cols {chunk}: gradient normwise error {r['g_rel']:.3e}")


# ---------------------------------------------------------------------------------------------------- buffers at offsets
def _offset_view(torch, src, off):
    """A contiguous copy of `src` that starts `off` floats into a larger allocation."""
    buf = torch.empty(src.numel() + off, dtype=torch.float32, device=src.device)
    v = buf[off:off + src.numel()].view(src.shape)
    v.copy_(src)
    return v


def _run(torch, cfg, feat, lab, call, lw=0.7):
    ctx = capi.Context(cfg)
    try:
        g = torch.full(tuple(feat.shape), float("nan"), dtype=torch.float32, device=feat.device)
        if call == "separate":
            tops = ctx.forward(feat, lab)
            ctx.backward(lw, g)
        else:
            tops = ctx.forward_backward(feat, lab, lw, g)
        torch.cuda.synchronize()
    finally:
        ctx.close()
    return np.array(tops, np.float32), g.cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("normalize_input", [0, 1])
@pytest.mark.parametrize("call", ["separate", "forward_backward"])
@pytest.mark.parametrize("Q,D", [(999, 101), (256, 128)])
def test_offset_inputs(cuda, Q, D, call, normalize_input):
    """Features and labels 1, 2 and 3 floats into larger allocations: every kernel that reads them falls back to scalar loads
    (operand preparation, operand split, L2 normalisation, the label sweeps; the LOCAL select runs its warp-per-row kernel), and tops
    and gradient are bit for bit those of 16-byte aligned copies."""
    torch = cuda
    x, lab = _inputs(Q, D, seed=Q + 3 * D)
    if normalize_input:
        x = np.ascontiguousarray(x * np.linspace(0.5, 3.0, Q, dtype=np.float32)[:, None])    # raw embeddings of varied norm
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    for name in ("usage", "local_rel"):
        cfg = capi.make_config(Q, D, normalize_input=normalize_input, **MININGS[name])
        t0, g0 = _run(torch, cfg, xt, lt, call)
        assert np.isfinite(g0).all() and np.abs(g0).max() > 0, name
        for off in (1, 2, 3):
            xv, lv = _offset_view(torch, xt, off), _offset_view(torch, lt, off)
            assert xv.data_ptr() % 16 and lv.data_ptr() % 16
            t1, g1 = _run(torch, cfg, xv, lv, call)
            tag = f"{name} Q{Q} D{D} {call} normalize_input={normalize_input} offset {off}"
            assert np.array_equal(_bits(t1), _bits(t0)), f"{tag}: tops {t1} vs {t0}"
            assert np.array_equal(_bits(g1), _bits(g0)), f"{tag}: gradient differs by up to {np.abs(g1 - g0).max():.3e}"


@pytest.mark.parametrize("Q,D", [(999, 101), (256, 128)])
def test_offset_outputs(cuda, Q, D):
    """A gradient output 1-3 floats off the 16-byte grid is refused with NPAIR_E_ARG by every backward entry point, and the context
    keeps working; one 16 bytes into an allocation gets the aligned result bit for bit."""
    torch = cuda
    x, lab = _inputs(Q, D, seed=Q + 5 * D)
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    cfg = capi.make_config(Q, D, **synth.USAGE_MINING)
    t0, g0 = _run(torch, cfg, xt, lt, "separate")

    def out_view(off, rows=Q):
        buf = torch.full((rows * D + 4,), float("nan"), dtype=torch.float32, device="cuda")
        return buf[off:off + rows * D].view(rows, D)

    def refused(fn):
        with pytest.raises(capi.NpairError) as e:
            fn()
        assert e.value.code == -1 and "16-byte aligned" in str(e.value), str(e.value)

    ctx = capi.Context(cfg)
    try:
        ctx.forward(xt, lt)
        for off in (1, 2, 3):
            bad = out_view(off)
            refused(lambda: ctx.backward(0.7, bad))
            refused(lambda: ctx.backward_partial(0.7, bad, None))
            refused(lambda: ctx.forward_backward(xt, lt, 0.7, bad))
            torch.cuda.synchronize()
            assert torch.isnan(bad).all(), "a refused call wrote its output"
        for off in (0, 4):                          # 16 bytes into the allocation: aligned
            g = out_view(off)
            ctx.backward(0.7, g)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(g.cpu().numpy()), _bits(g0)), f"backward at offset {off}"
            g = out_view(off)
            t = ctx.forward_backward(xt, lt, 0.7, g)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(np.array(t, np.float32)), _bits(t0)) and np.array_equal(_bits(g.cpu().numpy()), _bits(g0)), off
    finally:
        ctx.close()


@pytest.mark.parametrize("bwd_exchange", [0, 1])
def test_offset_outputs_emulated_ranks(cuda, bwd_exchange):
    """world 2: npair_backward_gathered (row-record form) and both outputs of npair_backward_partial (reduce-scatter form) refuse an
    unaligned output, and the same context then computes the gradient it computes without the refused call."""
    torch = cuda
    from gpu_harness import gpu_step_world
    Q, world, D = 333, 2, 101
    x, lab = _inputs(Q * world, D, seed=91)
    ref = gpu_step_world(x, lab, Q, world, synth.USAGE_MINING, FP16X2, TC, loss_weight=0.7, bwd_exchange=bwd_exchange)
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()

    def out_view(off, rows):
        buf = torch.full((rows * D + 4,), float("nan"), dtype=torch.float32, device="cuda")
        return buf[off:off + rows * D].view(rows, D)

    ctxs = [capi.Context(capi.make_config(Q, D, world=world, rank=r, bwd_exchange=bwd_exchange, **synth.USAGE_MINING)) for r in range(world)]
    try:
        for c in ctxs:
            c.forward_gathered(xt, lt)
        mode = ctxs[0].bwd_exchange_mode()
        assert mode == ref["mode"] == (2 if bwd_exchange == 0 else 1)
        local = torch.zeros((Q * world, D), dtype=torch.float32, device="cuda")
        total = torch.zeros_like(local)
        if mode == 2:
            rs = torch.empty((world, Q, 8), dtype=torch.float32, device="cuda")
            for r, c in enumerate(ctxs):
                c.row_scalars(rs[r])
        for r, c in enumerate(ctxs):
            for off in (1, 2, 3):
                if mode == 2:
                    with pytest.raises(capi.NpairError) as e:
                        c.backward_gathered(0.7, rs, out_view(off, Q))
                    assert e.value.code == -1
                else:
                    for lh, th in ((out_view(off, Q), out_view(0, Q * world)), (out_view(0, Q), out_view(off, Q * world))):
                        with pytest.raises(capi.NpairError) as e:
                            c.backward_partial(0.7, lh, th)
                        assert e.value.code == -1
            lh = out_view(4, Q)
            if mode == 2:
                c.backward_gathered(0.7, rs, lh)
            else:
                th = out_view(4, Q * world)
                c.backward_partial(0.7, lh, th)
                total += th
            local[r * Q:(r + 1) * Q] = lh
        torch.cuda.synchronize()
    finally:
        for c in ctxs:
            c.close()
    assert np.array_equal(_bits((local + total).cpu().numpy()), _bits(ref["dx"]))


# ---------------------------------------------------------------------------------------------------- tiny batches
@pytest.mark.parametrize("mining_name", ["default", "usage", "global_hard"])
@pytest.mark.parametrize("D", [1, 8])
@pytest.mark.parametrize("Q", [2, 3])
def test_tiny_batches(cuda, oracle, Q, D, mining_name):
    """Two or three rows: no negative at all (Q = 2, one class), or a row without a positive (Q = 3).  Where the oracle refuses the
    batch the library refuses it with the same error; otherwise the usual parity."""
    from gpu_harness import check_parity, gpu_step_world
    mining = dict(synth.DEFAULT_MINING) if mining_name == "default" else MININGS[mining_name]
    x, lab = synth.make_inputs(Q, D, seed=10 * Q + D)
    try:
        oracle.step_world(x, lab, oracle.make_config(Q, D, faithful_sorts=0, **mining), 1.0)
    except oracle.OracleError as e:
        with pytest.raises(capi.NpairError) as ge:
            gpu_step_world(x, lab, Q, 1, mining, FP16X2, TC)
        assert ge.value.code == ORACLE_TO_NPAIR[e.code], (ge.value.code, e.code)
        print(Q, D, mining_name, f"refused: {ge.value}")
        return
    r = check_parity(oracle, x, lab, Q, 1, mining, FP16X2, TC, tag=f"tiny Q{Q} D{D} {mining_name}")
    print(Q, D, mining_name, r)
