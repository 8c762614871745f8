"""Shared helpers for the GPU parity tests: run the CUDA path through the C ABI and compare with the oracle.

Two-level parity (SURVEY.md section 7 "hard parts"): mining is discontinuous in S, so
  L1: the GPU similarity matrix vs. the oracle's (tolerance by operand precision), and
  L2: the oracle re-run on the GPU's OWN S (S_inject) must give the same thresholds / loss / tops / gradient.
"""
import numpy as np
import torch

from npairloss_b200 import capi
import sim_ref

# Level 1 holds S to sim_ref's rules: componentwise against the exact sum of the piece products the sweep forms, and against fp64
# within that plus the operand format's error.
# normwise relative gradient bound at level 2
G_TOL = {capi.PREC_FP32_BF16X3: 1e-5, capi.PREC_FP32_FP16X2: 1e-5, capi.PREC_BF16: 2e-2}


def gpu_step_world(x, lab, Q, world, mining, prec, backend, loss_weight=1.0, num_tops=5, want_grad=True, bwd_exchange=0, **cfg_extra):
    """Emulates every rank on one GPU through the external-collectives API (the test plays NCCL's role).
    Returns dict(tops[world,5], dx[N,D], S[N,N], posi[N], nega[N], mode)."""
    N, D = x.shape
    dev = torch.device("cuda:0")
    xt = torch.from_numpy(x).to(dev).contiguous()
    lt = torch.from_numpy(lab).to(dev).contiguous()
    tops = np.zeros((world, 5), dtype=np.float32)
    S = np.zeros((N, N), dtype=np.float32)
    posi = np.zeros(N, dtype=np.float32)
    nega = np.zeros(N, dtype=np.float32)
    local = torch.zeros((N, D), dtype=torch.float32, device=dev)
    total = torch.zeros((N, D), dtype=torch.float32, device=dev)
    ctxs = []
    try:
        for r in range(world):
            cfg = capi.make_config(Q, D, world=world, rank=r, num_tops=num_tops, sim_precision=prec, gemm_backend=backend,
                                   bwd_exchange=bwd_exchange, **mining, **cfg_extra)
            ctx = capi.Context(cfg)
            ctxs.append(ctx)
            tops[r] = ctx.forward_gathered(xt, lt)
            S[r * Q:(r + 1) * Q] = ctx.debug_read(0, Q * N).reshape(Q, N)
            posi[r * Q:(r + 1) * Q] = ctx.debug_read(1, Q)
            nega[r * Q:(r + 1) * Q] = ctx.debug_read(2, Q)
        mode = ctxs[0].bwd_exchange_mode()
        if want_grad:
            if mode == 2:       # row-scalar exchange: "all-gather" the [Q][8] records of every rank
                rs = torch.empty((world, Q, 8), dtype=torch.float32, device=dev)
                for r in range(world):
                    ctxs[r].row_scalars(rs[r])
                for r in range(world):
                    g = torch.full((Q, D), float("nan"), dtype=torch.float32, device=dev)
                    ctxs[r].backward_gathered(loss_weight, rs, g)
                    local[r * Q:(r + 1) * Q] = g
            else:
                for r in range(world):
                    lh = torch.full((Q, D), float("nan"), dtype=torch.float32, device=dev)
                    if world > 1:
                        th = torch.full((N, D), float("nan"), dtype=torch.float32, device=dev)
                        ctxs[r].backward_partial(loss_weight, lh, th)
                        total += th
                    else:
                        ctxs[r].backward_partial(loss_weight, lh, None)
                    local[r * Q:(r + 1) * Q] = lh
    finally:
        for c in ctxs:
            c.close()
    torch.cuda.synchronize()
    dx = (local + total).cpu().numpy() if want_grad else None
    return dict(tops=tops, dx=dx, S=S, posi=posi, nega=nega, mode=mode)


def check_parity(oracle, x, lab, Q, world, mining, prec, backend, loss_weight=1.0, num_tops=5, tag="", bwd_exchange=0, gpu=None,
                 **cfg_extra):
    """gpu: a result of gpu_step_world with these arguments, to check instead of running the step again."""
    N, D = x.shape
    g = gpu if gpu is not None else gpu_step_world(x, lab, Q, world, mining, prec, backend, loss_weight, num_tops,
                                                   bwd_exchange=bwd_exchange, **cfg_extra)
    if g["mode"] != 1:
        # single-rank symmetric tiles / row-scalar exchange both rely on a bitwise symmetric similarity matrix
        assert np.array_equal(g["S"], g["S"].T), f"{tag} S is not bitwise symmetric (mode {g['mode']})"
    cfg = oracle.make_config(Q, D, world=world, num_tops=num_tops, faithful_sorts=0, **mining)
    # ---- level 1: similarities ----
    bad, m = sim_ref.check(g["S"], x, x, prec, "simt" if backend == capi.GEMM_SIMT_CHECK else "tc")
    assert not bad, f"{tag} L1 S: {bad} ({m})"
    # ---- level 2: oracle on the GPU's own S ----
    tops_o, dx_o = oracle.step_world(x, lab, cfg, loss_weight, S_inject_all=g["S"])
    for r in range(world):
        _, st = oracle.forward(x, lab, oracle.make_config(Q, D, world=world, rank=r, num_tops=num_tops, faithful_sorts=0, **mining),
                               S_inject=g["S"][r * Q:(r + 1) * Q])
        np.testing.assert_array_equal(g["posi"][r * Q:(r + 1) * Q], st["posi_thr"], err_msg=f"{tag} posi_thr rank {r}")
        np.testing.assert_array_equal(g["nega"][r * Q:(r + 1) * Q], st["nega_thr"], err_msg=f"{tag} nega_thr rank {r}")
    # loss: 1e-5 relative (north star); retrieval counters: discrete, allow one expf-rounding tie flip per 1000 rows
    np.testing.assert_allclose(g["tops"][:, 0], tops_o[:, 0], rtol=1e-5, atol=1e-6, err_msg=f"{tag} loss")
    n_ret = max(0, num_tops - 2)
    if n_ret:
        d = np.abs(g["tops"][:, 1:1 + n_ret] - tops_o[:, 1:1 + n_ret]) * Q
        assert d.max() <= max(1.0, Q / 1000.0) + 1e-3, f"{tag} retrieval counters differ by {d.max()} rows"
    np.testing.assert_allclose(g["tops"][:, num_tops - 1], tops_o[:, num_tops - 1], rtol=2e-6, err_msg=f"{tag} asum")
    gn = float(np.linalg.norm(dx_o))
    ge = float(np.linalg.norm(g["dx"] - dx_o))
    assert np.isfinite(g["dx"]).all(), f"{tag} non-finite gradient"
    assert ge <= G_TOL[prec] * max(gn, 1e-20), f"{tag} gradient normwise error {ge / max(gn, 1e-20):.3e}"
    return dict(s_ratio=m["ratio"], g_rel=ge / max(gn, 1e-20), loss=float(g["tops"][0, 0]))
