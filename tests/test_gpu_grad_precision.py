"""The gradient on the GPU against fp64, componentwise, per row and normwise (grad_ref.py), on the GPU's own S.

gpu_harness.check_parity holds the gradient to 1e-5 of the whole Q x D matrix's norm on well-spread rows.  Here every gradient path
is also held, element by element, to tau * B, where B is the magnitude of the terms the weight builder and the GEMM summed, and row
by row to the row's own 1e-5 or a multiple of the error of an fp32 SGEMM over the same weights, whichever is larger (grad_ref.tau and
grad_ref.SGEMM_FACTOR give the bounds and the values measured against them).  The inputs include rows
in a narrow cone (pairwise cosine up to 0.9996), where a row's weights are nearly equal and their rounding errors do not cancel, and
planted duplicate rows, which put many pairs exactly at the mining thresholds."""
import numpy as np
import pytest

from npairloss_b200 import capi, synth
import grad_ref
from grad_ref import SGEMM_FACTOR, U24
from gpu_harness import G_TOL, gpu_step_world

from grad_ref import FP16X2, BF16X3, BF16

pytestmark = pytest.mark.gpu

TC, SIMT = capi.GEMM_TCGEN05, capi.GEMM_SIMT_CHECK
NAME = {FP16X2: "fp16x2", BF16X3: "bf16x3", BF16: "bf16"}

HARD_HARD = dict(synth.DEFAULT_MINING, ap_method=synth.HARD, an_method=synth.HARD, margin_diff=-0.02)
GLOBAL_REL = dict(margin_ident=0.01, margin_diff=-0.02, identsn=-0.4, diffsn=-0.3, ap_region=synth.GLOBAL, ap_method=synth.RELATIVE_HARD,
                  an_region=synth.GLOBAL, an_method=synth.RELATIVE_HARD)
MININGS = {"rand": synth.DEFAULT_MINING, "usage": synth.USAGE_MINING, "hard": HARD_HARD, "global_rel": GLOBAL_REL}


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _inputs(kind, N, D, seed):
    if kind == "synth":
        return synth.make_inputs(N, D, seed, noise=2.5)
    if kind == "dup":                       # cosine ~0.99 cone of groups of four equal rows: ties at every threshold
        return grad_ref.cone_inputs(N, D, 0.1, seed, dup=4)
    return grad_ref.cone_inputs(N, D, float(kind), seed)


def _check(dx, ref, prec, path, tag, kind, N, chunk_cols=0):
    clustered = kind not in ("synth", "1")
    k = SGEMM_FACTOR["accumulator" if clustered or path == "split" else "spread"]
    # bf16 pieces carry 2^-9 of B per product, up to 15 % of R on clustered rows, where only the componentwise rule says anything.
    # The split GEMM accumulates all N columns in one accumulator (no chunks): 2.0e-5 .. 2.7e-5 normwise and up to 4.7e-5 of a row's
    # norm at N = 8192 on well-spread rows, measured on an H100 80GB HBM3 (700 W) with and without the weight scale alike
    rel = 0.5 if prec == BF16 and clustered else (max(G_TOL[prec], 2e-4) if path == "split" else G_TOL[prec])
    bad, m = grad_ref.violations(dx, ref, grad_ref.tau(prec, path, N, chunk_cols), rel=rel, k_sgemm=k)
    print(f"{tag} {NAME[prec]} {path}: normwise {m['normwise']:.2e} (sgemm {m['sgemm']:.2e}) worst row {m['row']:.3f} of its allowance, "
          f"componentwise {m['comp']:.1f} x 2^-24 of B")
    assert not bad, f"{tag} {NAME[prec]} {path}: " + "; ".join(bad)


def _world(x, lab, Q, world, mining, prec, path, kind, tag="", backend=TC, **cfg):
    flags = capi.FLAG_NO_FUSED_GRAD if path == "split" and world == 1 else 0
    g = gpu_step_world(x, lab, Q, world, mining, prec, backend, flags=flags, num_tops=2, **cfg)
    _check(g["dx"], grad_ref.step(x, lab, Q, world, g["S"], **mining), prec, path, f"{kind} {tag}", kind, Q * world,
           cfg.get("grad_chunk_cols", 0))


# ------------------------------------------------------------------------------------------------- world 1: inputs x minings
@pytest.mark.parametrize("path", ["fused", "split"])
@pytest.mark.parametrize("mining", list(MININGS))
@pytest.mark.parametrize("kind", ["synth", "1", "0.1", "0.02", "dup"])
def test_world1_fp16x2(torch, kind, mining, path):
    """Q = N = 1000, ragged D = 200."""
    x, lab = _inputs(kind, 1000, 200, 11)
    _world(x, lab, 1000, 1, MININGS[mining], FP16X2, path, kind, mining)


@pytest.mark.parametrize("path", ["fused", "split"])
@pytest.mark.parametrize("mining", ["rand", "usage"])
@pytest.mark.parametrize("kind", ["synth", "0.02"])
def test_world1_headline_shape(torch, kind, mining, path):
    """Q = N = 8192, D = 512: the flagship step's shape."""
    x, lab = _inputs(kind, 8192, 512, 12)
    _world(x, lab, 8192, 1, MININGS[mining], FP16X2, path, kind, f"{mining} 8192")


@pytest.mark.parametrize("prec", [BF16X3, BF16])
@pytest.mark.parametrize("path", ["fused", "split"])
@pytest.mark.parametrize("kind", ["synth", "0.02", "dup"])
def test_world1_other_formats(torch, kind, path, prec):
    x, lab = _inputs(kind, 1000, 200, 13)
    _world(x, lab, 1000, 1, MININGS["rand"], prec, path, kind)


@pytest.mark.parametrize("prec", [FP16X2, BF16X3])
@pytest.mark.parametrize("kind", ["synth", "0.1", "dup"])
def test_simt_cross_check(torch, kind, prec):
    x, lab = _inputs(kind, 384, 72, 14)
    _world(x, lab, 384, 1, MININGS["usage"], prec, "simt", kind, backend=SIMT)


@pytest.mark.parametrize("chunk", [256, 0, -1])
@pytest.mark.parametrize("kind", ["synth", "0.02"])
def test_grad_chunk_cols(torch, kind, chunk):
    x, lab = _inputs(kind, 4096, 256, 15)
    _world(x, lab, 4096, 1, MININGS["rand"], FP16X2, "fused", kind, f"chunk {chunk}", grad_chunk_cols=chunk)


@pytest.mark.parametrize("kind", ["synth", "0.1"])
def test_split_k_heavy_shape(torch, kind):
    """Q = 999, D = 101 (test_gpu_ragged_shapes.SPLITK_SHAPES): a few 128 x 256 tiles, K split over many slices."""
    x, lab = _inputs(kind, 999, 101, 16)
    _world(x, lab, 999, 1, MININGS["rand"], FP16X2, "fused", kind)


# --------------------------------------------------------------------------------------------------- emulated ranks
@pytest.mark.parametrize("bwd_exchange", [0, 1], ids=["records", "reduce_scatter"])
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("kind", ["synth", "0.02"])
def test_emulated_world(torch, kind, world, bwd_exchange):
    """Rows of world - 1 other ranks get 1/world of their transposed weight: the row-record exchange folds it into the fused kernel's
    column term, the reduce-scatter form into the alpha of its transposed GEMM."""
    Q = 2048 // world
    x, lab = _inputs(kind, Q * world, 128, 17)
    _world(x, lab, Q, world, MININGS["rand"], FP16X2, "split" if bwd_exchange else "fused", kind, f"w{world}",
           bwd_exchange=bwd_exchange)


# --------------------------------------------------------------------------------------------------- row-block mode
@pytest.mark.parametrize("kind", ["synth", "0.02"])
def test_row_blocks(torch, kind):
    """Three blocks of 384 rows.  Row-block mode keeps no S to read; its gradient is that of the materialised path on the same S."""
    Q, D = 1024, 192
    x, lab = _inputs(kind, Q, D, 18)
    mining = MININGS["rand"]
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    out = {}
    for rows in (0, 384):
        ctx = capi.Context(capi.make_config(Q, D, num_tops=2, sim_block_rows=rows, **mining))
        try:
            ctx.forward(xt, lt)
            dx = torch.full_like(xt, float("nan"))
            ctx.backward(1.0, dx)
            torch.cuda.synchronize()
            out[rows] = dx.cpu().numpy()
            if rows == 0:
                S = ctx.debug_read(0, Q * Q).reshape(Q, Q)
        finally:
            ctx.close()
    _check(out[384], grad_ref.step(x, lab, Q, 1, S, **mining), FP16X2, "fused", f"{kind} row blocks", kind, Q)


# --------------------------------------------------------------------------------------------------- cross-batch memory
@pytest.mark.parametrize("path", ["fused", "split"])
@pytest.mark.parametrize("Q,m", [(1024, 16384), (512, 57344)])
def test_memory_step(torch, Q, m, path):
    """dx = (1/2)(lw/Q)(G . X_total + G[:, 0:Q]^T . x) on cone rows (cosine ~0.99) whose memory shares the batch's classes."""
    D = 128
    x, lab = grad_ref.cone_inputs(Q + m, D, 0.1, 19)
    lab = np.concatenate([lab[:Q], lab[Q:] % (Q // 2)]).astype(np.float32)      # the memory rows fall into the batch's classes
    mining = MININGS["usage"]
    flags = capi.FLAG_NO_FUSED_GRAD if path == "split" else 0
    xt, lt, xm, lm = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x[:Q], lab[:Q], x[Q:], lab[Q:]))
    ctx = capi.Context(capi.make_config(Q, D, num_tops=2, flags=flags, **mining), memory_rows=m)
    try:
        ctx.forward_memory(xt, lt, xm, lm, m)
        dx = torch.full_like(xt, float("nan"))
        ctx.backward(1.0, dx)
        torch.cuda.synchronize()
        S = ctx.debug_read(0, Q * (Q + m)).reshape(Q, Q + m)
    finally:
        ctx.close()
    ref = grad_ref.step(x, lab, Q, 1, S, **mining)
    ref = {k: ref[k][:Q] for k in ("R", "B", "R32")}                            # the anchors' rows
    _check(dx.cpu().numpy(), ref, FP16X2, path, f"memory Q {Q} m {m}", "0.1", Q + m)
