"""The memory rows' gradient (DESIGN 4.6) without a GPU: the fp64 reference (rows [Q, N) of grad_ref.step over [x; y]) against the C++
oracle's world-W backward it must equal at m = (W - 1) Q, against finite differences of the loss, its anchor weighting, the exported
symbols and the torch API's checks and plumbing."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import grad_ref
from npairloss_b200 import capi, synth, torch_api
from oracle import npair_oracle_np as onp

ALL_MINING = [dict(margin_ident=0.02, margin_diff=-0.03, identsn=-0.4, diffsn=-0.3, ap_region=apR, ap_method=apM, an_region=anR,
                   an_method=anM)
              for apR, apM, anR, anM in itertools.product([0, 1], [0, 1, 2, 3, 4], [0, 1], [0, 1, 2, 3, 4])]


def _mem_grad(x, l, y, ly, w=None, **kw):
    """d_mem_diff in fp64 [m, D]: rows [Q, N) of grad_ref.step over the database [x; y]."""
    Q = x.shape[0]
    return grad_ref.step(np.concatenate([x, y]), np.concatenate([l, ly]), Q, 1, None, w, **kw)["R"][Q:]


def _unit_rows(n, D, rng):
    x = rng.standard_normal((n, D))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("W", [2, 3])
def test_reference_is_w_times_the_world_oracles_total_half(oracle, W):
    """At m = (W - 1) Q the memory rows are ranks 1 .. W-1 of a world-W step on [x; y]: their gradient is W times rank 0's addend of
    the all-reduce, d_total_half[Q:] (the C++ oracle's own fp32 total_diff of npo_backward_partial with the blend's 1/2 and 1/world),
    for all 100 mining combinations."""
    Q, D = 24, 16
    xt, lt = synth.make_inputs(W * Q, D, seed=40 + W, imgs_per_class=3, noise=0.7)
    L = oracle.lib()
    fp = C.POINTER(C.c_float)
    assert len(ALL_MINING) == 100
    for kw in ALL_MINING:
        cfg = oracle.make_config(Q, D, world=W, rank=0, **kw)
        _, st = oracle.forward(xt, lt, cfg)
        lh = np.zeros((Q, D), dtype=np.float32)
        th = np.zeros((W * Q, D), dtype=np.float32)
        assert L.npo_backward_partial(C.byref(cfg), xt.ctypes.data_as(fp), C.byref(st["_st"]), C.c_float(0.7), lh.ctypes.data_as(fp),
                                      th.ctypes.data_as(fp)) == 0
        total_half = 0.5 / W * th.astype(np.float64)          # the blend's 1/2 and 1/world (.cu:474, :492-497): d_total_half
        want = W * total_half[Q:]
        got = _mem_grad(xt[:Q], lt[:Q], xt[Q:], lt[Q:], loss_weight=0.7, **kw)
        assert np.linalg.norm(got - want) <= 2e-6 * max(np.linalg.norm(want), 1e-12), kw


def _fd_inputs(seed, Q=10, m=7, D=6):
    rng = np.random.default_rng(seed)
    x, y = _unit_rows(Q, D, rng), _unit_rows(m, D, rng)
    l = (np.arange(Q) % 4).astype(np.float32)
    ly = np.array([0, 1, 2, 3, 5, 1, 2][:m], dtype=np.float32)     # label 5: no anchor of that class
    return x, l, y, ly


def _loss(x, l, y, ly, w=None, **mining):
    """The step's loss in fp64 as a function of the memory rows y (S = x . [x; y]^T in fp64, the forward's selections and maxima
    evaluated in fp64 too): what finite differences with respect to y differentiate.  Weighted: -(1/Q) sum_i w_i log(A_i / T_i)."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    Q = x.shape[0]
    _, st = onp_forward(x.astype(np.float32), l, y.astype(np.float32), ly, **mining)
    sel1 = st["temp1"] > 0                                      # the forward's selections, held fixed
    sel2 = st["temp2"] > 0
    S = x @ np.concatenate([x, y]).T
    E = np.exp(S - st["max_all"].astype(np.float64)[:, None])
    A = np.where(sel1, E, 0.0).sum(axis=1)
    T = A + np.where(sel2, E, 0.0).sum(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        lv = np.where(A > 0, np.log(A / T), 0.0)
    wv = np.ones(Q) if w is None else np.asarray(w, dtype=np.float64)
    return -(wv * lv).sum() / Q


def _fd(x, l, y, ly, w=None, h=1e-5, **mining):
    g = np.zeros(y.shape)
    y64 = y.astype(np.float64)
    for p, d in itertools.product(range(y.shape[0]), range(y.shape[1])):
        e = np.zeros_like(y64)
        e[p, d] = h
        g[p, d] = (_loss(x, l, y64 + e, ly, w, **mining) - _loss(x, l, y64 - e, ly, w, **mining)) / (2 * h)
    return g


@pytest.mark.parametrize("mining", [dict(), dict(ap_method=onp.HARD, an_method=onp.HARD, margin_diff=-0.05),
                                    dict(an_method=onp.EASY, margin_diff=0.1)])
def test_reference_is_half_the_gradient_of_the_loss(mining):
    """2 d_mem_diff is the gradient of the loss with respect to the memory rows (central differences, the selections held fixed: the
    test asserts that no perturbation moves a pair across its threshold)."""
    x, l, y, ly = _fd_inputs(3)
    _, st = onp_forward(x, l, y, ly, **mining)
    for s in (-1e-5, 1e-5):                                 # the selections of the perturbed steps are the unperturbed one's
        _, st2 = onp_forward(x, l, y + np.float32(s), ly, **mining)
        assert np.array_equal(st["temp1"] > 0, st2["temp1"] > 0) and np.array_equal(st["temp2"] > 0, st2["temp2"] > 0), mining
    got = 2 * _mem_grad(x, l, y, ly, **mining)
    fd = _fd(x, l, y, ly, **mining)
    assert np.abs(got).max() > 1e-3
    np.testing.assert_allclose(got, fd, rtol=2e-4, atol=2e-6)


def onp_forward(x, l, y, ly, **mining):
    return onp.forward(np.concatenate([x, y]), np.concatenate([l, ly]), x.shape[0], num_tops=2, **mining)


def test_weighted_reference_is_linear_in_w_and_matches_the_weighted_loss():
    x, l, y, ly = _fd_inputs(9)
    Q = x.shape[0]
    w = np.array([1.0, 0.0, 0.5, 0.25, 1.0, 0.0, 0.75, 0.125, 1.0, 0.3], dtype=np.float32)
    d = _mem_grad(x, l, y, ly, w=w)
    # linear in w: the sum of each anchor's share
    parts = sum(w[i] * _mem_grad(x, l, y, ly, w=np.eye(Q, dtype=np.float32)[i]) for i in range(Q))
    np.testing.assert_allclose(d, parts, rtol=1e-12, atol=1e-15)
    # anchors with w = 0 contribute nothing: their weights rows are exactly 0
    G, _ = grad_ref.step(np.concatenate([x, y]), np.concatenate([l, ly]), Q, 1, None, w)["G"][0]
    assert not G[w == 0].any()
    np.testing.assert_allclose(d, 0.5 * G[w > 0, Q:].T @ x[w > 0].astype(np.float64), rtol=1e-12, atol=1e-15)
    # and twice it is the gradient of the weighted loss
    np.testing.assert_allclose(2 * d, _fd(x, l, y, ly, w), rtol=2e-4, atol=2e-6)
    # w = 1 is the unweighted reference
    np.testing.assert_array_equal(_mem_grad(x, l, y, ly, w=np.ones(Q, np.float32)), _mem_grad(x, l, y, ly))


def test_symbols_are_exported_and_refuse_without_a_context():
    L = capi.lib()
    for sym in ("npair_backward_memory", "npair_backward_memory_device_weight"):
        assert sym in capi.EXPORTS and hasattr(L, sym), sym
    assert L.npair_backward_memory(None, C.c_float(1.0), None, None, None) == -1
    assert L.npair_backward_memory_device_weight(None, None, None, None, None) == -1


# ---- torch API: checks and plumbing with a stand-in context ----
class FakeMemoryContext:
    def __init__(self, cfg, nccl_id, log):
        self.cfg, self.calls = cfg, log

    def forward_memory(self, feat, label, rows, labels, m):
        self.calls.append(("fwd_mem", tuple(feat.shape), tuple(rows.shape), labels.dtype, m))
        return [1.5, 0.5, 0.5, 0.5, 1.0]

    def forward(self, feat, label):
        self.calls.append(("fwd",))
        return [1.5, 0.5, 0.5, 0.5, 1.0]

    def backward(self, lw, diff):
        self.calls.append(("bwd", lw))
        diff.fill_(lw)

    def backward_memory(self, lw, diff, mem_diff):
        self.calls.append(("bwd_mem", lw, tuple(mem_diff.shape)))
        diff.fill_(lw)
        mem_diff.fill_(3.0 * lw)


def _module(**kw):
    log, made = [], []

    def factory(cfg, nid):
        made.append(FakeMemoryContext(cfg, nid, log))
        return made[-1]
    return torch_api.NPairLoss(_context_factory=factory, **kw), log, made


def test_torch_extra_rows_plumbing():
    mod, log, made = _module(true_gradient=True)
    x = torch.randn(6, 4, requires_grad=True)
    proxies = torch.randn(3, 4, requires_grad=True)
    loss, _ = mod(x, torch.tensor([0, 0, 1, 1, 2, 2]), extra_rows=proxies, extra_labels=torch.arange(3))
    (2.0 * loss).backward()
    assert log[0] == ("fwd_mem", (6, 4), (3, 4), torch.float32, 3)
    assert log[1] == ("bwd_mem", 2.0, (3, 4))
    np.testing.assert_array_equal(x.grad.numpy(), np.full((6, 4), 4.0, np.float32))          # true_gradient doubles both
    np.testing.assert_array_equal(proxies.grad.numpy(), np.full((3, 4), 12.0, np.float32))
    # rows without requires_grad: the plain backward
    mod(x, torch.tensor([0, 0, 1, 1, 2, 2]), extra_rows=proxies.detach(), extra_labels=torch.arange(3))[0].backward()
    assert log[-1] == ("bwd", 1.0)
    # the capacity only grows: more rows re-create the context, fewer keep it
    assert len(made) == 1
    mod(x, torch.zeros(6), extra_rows=torch.randn(5, 4), extra_labels=torch.arange(5))
    assert len(made) == 2
    mod(x, torch.zeros(6), extra_rows=torch.randn(2, 4), extra_labels=torch.arange(2))
    assert len(made) == 2


def test_torch_extra_rows_argument_checks():
    x, lab = torch.randn(6, 4), torch.zeros(6)
    rows, rl = torch.randn(3, 4), torch.arange(3)
    mod, _, made = _module()
    for kw, err in ((dict(extra_rows=rows), ValueError), (dict(extra_labels=rl), ValueError),
                    (dict(extra_rows=rows.double(), extra_labels=rl), TypeError),
                    (dict(extra_rows=[[0.0] * 4], extra_labels=rl), TypeError),
                    (dict(extra_rows=torch.randn(3, 5), extra_labels=rl), ValueError),
                    (dict(extra_rows=torch.randn(3), extra_labels=rl), ValueError),
                    (dict(extra_rows=rows, extra_labels=torch.arange(4)), ValueError),
                    (dict(extra_rows=rows, extra_labels=torch.zeros(3, 1)), ValueError),
                    (dict(extra_rows=rows.to("meta"), extra_labels=rl), ValueError),
                    (dict(extra_rows=rows, extra_labels=rl.to("meta")), ValueError),
                    (dict(extra_rows=rows, extra_labels=torch.tensor([0.5, 1.0, 2 ** 25 + 1], dtype=torch.float64)), ValueError)):
        with pytest.raises(err):
            mod(x, lab, **kw)
    assert not made                                          # refused before any context exists
    with pytest.raises(ValueError, match="memory_rows"):
        _module(memory_rows=8)[0](x, lab, extra_rows=rows, extra_labels=rl)
    with pytest.raises(ValueError, match="world"):
        _module(world=2)[0](x, lab, extra_rows=rows, extra_labels=rl)


def test_torch_extra_rows_refuse_what_a_memory_context_refuses():
    """Configurations a memory context does not support are refused before any context exists, with ValueError."""
    x, lab = torch.randn(6, 4), torch.zeros(6)
    rows, rl = torch.randn(3, 4), torch.arange(3)
    for kw in (dict(global_scope=1), dict(sim_block_rows=128), dict(flags=capi.sim_block_flags(256)),
               dict(gemm_backend=capi.GEMM_SIMT_CHECK)):
        mod, _, made = _module(**kw)
        with pytest.raises(ValueError, match="cross-batch memory"):
            mod(x, lab, extra_rows=rows, extra_labels=rl)
        assert not made, kw
    mod, log, made = _module(flags=capi.FLAG_NO_FUSED_GRAD)
    with pytest.raises(ValueError, match="FLAG_NO_FUSED_GRAD"):
        mod(x, lab, extra_rows=rows.clone().requires_grad_(True), extra_labels=rl)
    mod(x, lab, extra_rows=rows, extra_labels=rl)               # no gradient wanted: the forward runs
    assert log[-1][0] == "fwd_mem"


def test_capi_last_m_follows_the_last_forward():
    """backward_memory sizes mem_diff by the last forward's m; a non-memory forward resets it (no device needed: the stand-in library
    returns OK for every call)."""
    class Lib:
        def __getattr__(self, name):
            return lambda *a: 0
    ctx = capi.Context.__new__(capi.Context)
    ctx.cfg, ctx._h, ctx.last_m = capi.make_config(6, 4), C.c_void_p(), 0
    old = capi._LIB
    capi._LIB = Lib()
    try:
        ctx.forward_memory_ptr(1, 2, 3, 4, 5)
        assert ctx.last_m == 5
        ctx.forward_ptr(1, 2)
        assert ctx.last_m == 0
    finally:
        capi._LIB = old

