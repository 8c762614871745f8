"""Cross-batch memory (DESIGN 4.3) without a GPU: the NumPy oracle's memory step against the C++ oracle's world-W step it must equal
at m = (W - 1) Q, the workspace sizes, the exported symbols and the host-side argument checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from npairloss_b200 import capi
from oracle import npair_oracle_np as onp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MINING = [dict(), dict(ap_method=onp.HARD, an_method=onp.HARD, margin_diff=-0.05),
          dict(ap_region=onp.GLOBAL, ap_method=onp.RELATIVE_HARD, identsn=0.5, an_region=onp.GLOBAL, an_method=onp.HARD),
          dict(an_method=onp.RELATIVE_HARD, diffsn=-0.3, ap_method=onp.EASY)]


def _inputs(n, D, classes, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, D)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return x.astype(np.float32), rng.integers(0, classes, n).astype(np.float32)


@pytest.mark.parametrize("mining", MINING)
@pytest.mark.parametrize("W", [2, 3])
def test_memory_step_is_rank_0_of_a_world_step(oracle, mining, W):
    """At m = (W - 1) Q the memory step is rank 0 of a world-W step on [x; x_mem]: its tops, and its gradient rows 0 .. Q-1 rebuilt
    from rank 0's halves as d_local_half + W d_total_half.  The tops of the world-W step are the C++ oracle's."""
    Q, D = 24, 16
    xt, lt = _inputs(W * Q, D, 7, 11 + W)
    tops_w, _ = oracle.forward(xt, lt, oracle.make_config(Q, D, world=W, rank=0, **mining))
    _, st = onp.forward(xt, lt, Q, W, 0, **mining)                   # rank 0's weights, for the halves in fp64
    G = onp.grad_weights(st, Q, 1.5)
    local = 0.5 * (G @ xt.astype(np.float64))                        # d_local_half
    total = 0.5 / W * (G.T @ xt[:Q].astype(np.float64))              # rank 0's d_total_half
    tops_m, dx_m, _ = onp.step_world_fp64(xt, lt, Q, 1, 1.5, **mining)          # world 1 on [x; x_mem]
    tops_m, dx_m = tops_m[0], dx_m[:Q]
    np.testing.assert_array_equal(tops_m, tops_w)
    np.testing.assert_allclose(dx_m, local + W * total[:Q], rtol=1e-12, atol=1e-15)
    tops_all, _ = oracle.step_world(xt, lt, oracle.make_config(Q, D, world=W, **mining), 1.5)
    np.testing.assert_array_equal(tops_m, tops_all[0])


@pytest.mark.parametrize("mining", MINING)
def test_memory_step_without_memory_is_the_plain_step(oracle, mining):
    Q, D = 30, 12
    x, l = _inputs(Q, D, 6, 5)
    tops_p, dx_p = oracle.step_world(x, l, oracle.make_config(Q, D, **mining), 0.7)
    tops_m, dx_m, _ = onp.step_world_fp64(x, l, Q, 1, 0.7, **mining)
    np.testing.assert_array_equal(tops_m[0], tops_p[0])
    np.testing.assert_allclose(dx_m, dx_p, rtol=2e-6, atol=1e-9)


def _bytes(M, **kw):
    return capi.lib().npair_memory_workspace_bytes(C.byref(capi.make_config(kw.pop("Q", 256), kw.pop("D", 64), **kw)), M)


def test_memory_workspace_bytes():
    L = capi.lib()
    for kw in (dict(), dict(flags=capi.FLAG_NO_FUSED_GRAD), dict(normalize_input=1), dict(sim_precision=capi.PREC_BF16),
               dict(world=2), dict(gemm_backend=capi.GEMM_SIMT_CHECK), dict(global_scope=1)):
        cfg = capi.make_config(256, 64, **kw)
        assert L.npair_memory_workspace_bytes(C.byref(cfg), 0) == L.npair_workspace_bytes(C.byref(cfg)) > 0, kw
        assert capi.memory_workspace_bytes(cfg, 0) == L.npair_workspace_bytes(C.byref(cfg))
    for kw in (dict(), dict(flags=capi.FLAG_NO_FUSED_GRAD), dict(sim_precision=capi.PREC_FP32_BF16X3),
               dict(ap_region=capi.GLOBAL, ap_method=capi.RELATIVE_HARD, identsn=0.3)):
        sizes = [_bytes(M, **kw) for M in (0, 1, 37, 256, 1000, 8192, 65536)]
        assert all(a < b for a, b in zip(sizes, sizes[1:])), (kw, sizes)
    # refused: world > 1, row-block mode, SIMT, global_scope, negative capacity
    for kw in (dict(world=2), dict(sim_block_rows=128, Q=512), dict(gemm_backend=capi.GEMM_SIMT_CHECK), dict(global_scope=1)):
        assert _bytes(64, **kw) == 0, kw
    assert _bytes(-1) == 0


def test_memory_symbols_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "npair_b200.h")).read()
    L = capi.lib()
    for sym in ("npair_create_memory", "npair_memory_workspace_bytes", "npair_forward_memory"):
        assert re.search(r"\b%s\s*\(" % sym, hdr), sym
        assert hasattr(L, sym) and sym in capi.EXPORTS, sym


def test_memory_argument_checks_without_a_device():
    """Creation refuses the configurations a memory does not support before it looks for a device, and a forward without a context
    is refused."""
    L = capi.lib()
    for kw in (dict(world=2), dict(sim_block_rows=128, Q=512), dict(gemm_backend=capi.GEMM_SIMT_CHECK), dict(global_scope=1)):
        q = kw.pop("Q", 64)
        with pytest.raises(capi.NpairError) as e:
            capi.Context(capi.make_config(q, 32, **kw), memory_rows=128)
        assert e.value.code == -1, kw
    h = C.c_void_p()
    assert L.npair_create_memory(C.byref(capi.make_config(64, 32)), -5, C.byref(h)) == -1
    assert L.npair_create_memory(C.byref(capi.make_config(0, 32)), 16, C.byref(h)) == -1
    tops = (C.c_float * 5)()
    assert L.npair_forward_memory(None, None, None, None, None, 0, tops, None) == -1
    with pytest.raises(ValueError):
        from npairloss_b200.torch_api import NPairLoss
        NPairLoss(world=2, memory_rows=64)
