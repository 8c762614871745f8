"""The asynchronous training step and CUDA-graph capture (DESIGN 4.4) on the GPU: npair_forward_async / npair_forward_memory_async and
npair_backward_device_weight bit for bit against npair_forward + npair_backward, no host wait, device errors through
npair_async_status, capture and replay of whole steps (also interleaved with eager steps), the calls refused during a capture, and a
whole torch training step captured with torch.cuda.graph."""
import ctypes as C

import numpy as np
import pytest

from npairloss_b200 import capi, synth, torch_api

pytestmark = pytest.mark.gpu

FP16X2, BF16X3, BF16 = capi.PREC_FP32_FP16X2, capi.PREC_FP32_BF16X3, capi.PREC_BF16
E_ARG, E_EMPTY_LIST, E_POS_RANGE, E_STATE = -1, -4, -5, -6
LOSS_WEIGHTS = [1.0, 0.5, 1.3, 2.0 ** -20, 0.0, -1.0]
USAGE = dict(synth.USAGE_MINING)
LOCAL_SN = dict(ap_region=capi.LOCAL, ap_method=capi.RELATIVE_HARD, an_region=capi.LOCAL, an_method=capi.RELATIVE_HARD, identsn=-0.4,
                diffsn=-0.3, margin_diff=-0.02)
GLOBAL_SN = dict(LOCAL_SN, ap_region=capi.GLOBAL, an_region=capi.GLOBAL)
# about 50 ms of GPU time at the H100's clocks
SLEEP_CYCLES = 100_000_000


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0), "GPU tests need an H100"
    return torch


def _inputs(torch, Q, D, seed, per_class=2, noise=1.0):
    x, lab = synth.make_inputs(Q, D, seed=seed, imgs_per_class=per_class, noise=noise)
    return torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()


def _bits(t):
    return t.detach().cpu().numpy().view(np.uint32)


def _sync_step(torch, ctx, x, l, lw, mem=None):
    """npair_forward (or npair_forward_memory) + npair_backward: (tops [5] fp32, gradient) on the host."""
    tops = ctx.forward(x, l) if mem is None else ctx.forward_memory(x, l, *mem)
    dx = torch.full_like(x, float("nan"))
    ctx.backward(lw, dx)
    torch.cuda.synchronize()
    return np.array(tops, dtype=np.float32), dx.cpu().numpy()


def _async_step(torch, ctx, x, l, lw, mem=None):
    """npair_forward_async (or _memory_async) + npair_backward_device_weight, with the loss weight in device memory."""
    tops = torch.full((5,), 7.0, device="cuda")
    if mem is None:
        ctx.forward_async(x, l, tops)
    else:
        ctx.forward_memory_async(x, l, *mem, tops)
    dx = torch.full_like(x, float("nan"))
    ctx.backward_device_weight(torch.tensor([lw], dtype=torch.float32, device="cuda"), dx)
    torch.cuda.synchronize()
    return tops.cpu().numpy(), dx.cpu().numpy()


def _same(a, b, tag):
    np.testing.assert_array_equal(a[0].view(np.uint32), b[0].view(np.uint32), err_msg=f"{tag} tops")
    np.testing.assert_array_equal(a[1].view(np.uint32), b[1].view(np.uint32), err_msg=f"{tag} gradient")


# ---------------------------------------------------------------------------------------------------------- 1. bit for bit
CASES = {
    "fp16x2 usage": dict(Q=512, D=128),
    "bf16x3 usage": dict(Q=512, D=128, sim_precision=BF16X3),
    "bf16 usage": dict(Q=512, D=128, sim_precision=BF16),
    "local general SN": dict(Q=512, D=128, mining=LOCAL_SN),
    "global general SN": dict(Q=512, D=128, mining=GLOBAL_SN),
    "ragged": dict(Q=999, D=101, per_class=3),
    "normalize_input": dict(Q=512, D=128, normalize_input=1, noise=3.0),
    "row blocks": dict(Q=900, D=128, sim_block_rows=256),
    "memory m=0": dict(Q=384, D=96, memory=(300, 0)),
    "memory m=261": dict(Q=384, D=96, memory=(300, 261)),
    "memory m=261 normalize_input": dict(Q=384, D=96, memory=(300, 261), normalize_input=1, noise=3.0),
    "no fused gradient": dict(Q=512, D=128, flags=capi.FLAG_NO_FUSED_GRAD),
    "SIMT": dict(Q=256, D=64, gemm_backend=capi.GEMM_SIMT_CHECK),
}


def _case(torch, case, seed=11):
    """(config, memory capacity, x, labels, memory (rows, labels, m) or None) of a case of CASES / GRAPH_CASES"""
    kw = dict(case)
    Q, D = kw.pop("Q"), kw.pop("D")
    per_class, noise = kw.pop("per_class", 2), kw.pop("noise", 1.0)
    M, m = kw.pop("memory", (0, None))
    cfg = capi.make_config(Q, D, **kw.pop("mining", USAGE), **kw)
    x, l = _inputs(torch, Q + (m or 0), D, seed, per_class, noise)
    mem = None
    if m is not None:
        mem = (x[Q:].contiguous(), l[Q:].contiguous(), m)
        x, l = x[:Q].contiguous(), l[:Q].contiguous()
    return cfg, M, x, l, mem


@pytest.mark.parametrize("name", list(CASES))
def test_async_step_is_the_synchronous_step_bit_for_bit(torch, name):
    """Tops as packed fp32 and the gradient bit for bit, for every loss weight; the device-weight backward also after a synchronous
    forward."""
    cfg, M, x, l, mem = _case(torch, CASES[name])
    ref, ctx = capi.Context(cfg, memory_rows=M), capi.Context(cfg, memory_rows=M)
    try:
        for lw in LOSS_WEIGHTS:
            want = _sync_step(torch, ref, x, l, lw, mem)
            assert np.isfinite(want[0]).all() and np.isfinite(want[1]).all(), (name, lw)
            _same(_async_step(torch, ctx, x, l, lw, mem), want, f"{name} lw={lw} async")
            # synchronous forward, device-weight backward
            tops = ctx.forward(x, l) if mem is None else ctx.forward_memory(x, l, *mem)
            dx = torch.full_like(x, float("nan"))
            ctx.backward_device_weight(torch.tensor([lw], dtype=torch.float32, device="cuda"), dx)
            torch.cuda.synchronize()
            _same((np.array(tops, np.float32), dx.cpu().numpy()), want, f"{name} lw={lw} sync forward")
        ctx.async_status()
    finally:
        ref.close(); ctx.close()


@pytest.mark.parametrize("num_tops", [1, 2, 3, 4, 5])
def test_num_tops(torch, num_tops):
    """d_tops receives what tops_host would: the tops of num_tops, 0 after them."""
    cfg = capi.make_config(256, 64, num_tops=num_tops, **USAGE)
    x, l = _inputs(torch, 256, 64, 5)
    ref, ctx = capi.Context(cfg), capi.Context(cfg)
    try:
        want = _sync_step(torch, ref, x, l, 1.0)
        got = _async_step(torch, ctx, x, l, 1.0)
        _same(got, want, f"num_tops={num_tops}")
        assert (got[0][num_tops:] == 0).all()
    finally:
        ref.close(); ctx.close()


# ---------------------------------------------------------------------------------------------------------- 2. no host wait
def test_calls_return_before_the_gpu_reaches_them(torch):
    cfg = capi.make_config(512, 128, **USAGE)
    x, l = _inputs(torch, 512, 128, 21)
    ref, ctx = capi.Context(cfg), capi.Context(cfg)
    try:
        want = _sync_step(torch, ref, x, l, 0.5)
        _async_step(torch, ctx, x, l, 0.5)                   # loads the kernels
        tops, dx = torch.empty(5, device="cuda"), torch.empty_like(x)
        lw = torch.tensor([0.5], device="cuda")
        torch.cuda.synchronize()
        torch.cuda._sleep(SLEEP_CYCLES)
        ctx.forward_async(x, l, tops)
        ctx.backward_device_weight(lw, dx)
        ev = torch.cuda.Event()
        ev.record()
        assert not ev.query(), "the asynchronous calls waited for the GPU"
        torch.cuda.synchronize()
        _same((tops.cpu().numpy(), dx.cpu().numpy()), want, "behind a sleep")
    finally:
        ref.close(); ctx.close()


def test_npairloss_nonblocking_makes_no_synchronising_call(torch):
    x, l = _inputs(torch, 256, 64, 22)
    loss_fn = torch_api.NPairLoss(blocking=False, **USAGE)
    xr = x.clone().requires_grad_(True)
    loss_fn(xr, l)[0].backward()                             # creates the context
    torch.cuda.synchronize()
    xr.grad = None
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss, tops = loss_fn(xr, l)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    ref = torch_api.NPairLoss(**USAGE)
    xb = x.clone().requires_grad_(True)
    lb, tb = ref(xb, l)
    lb.backward()
    np.testing.assert_array_equal(_bits(tops), _bits(tb))
    np.testing.assert_array_equal(_bits(loss), _bits(lb))
    np.testing.assert_array_equal(_bits(xr.grad), _bits(xb.grad))
    loss_fn.async_status()


# ---------------------------------------------------------------------------------------------------------- 3. device errors
def test_device_errors_give_nan_tops_and_a_status(torch):
    Q, D = 16, 8
    x, l = _inputs(torch, Q, D, 1)
    for kw, labels, code in ((dict(ap_method=capi.RELATIVE_HARD), l, E_POS_RANGE),                      # identsn = -1: pos = -1
                             (dict(an_region=capi.GLOBAL, an_method=capi.HARD), torch.arange(Q, dtype=torch.float32, device="cuda"),
                              E_EMPTY_LIST)):                                                          # no positive pair
        cfg = capi.make_config(Q, D, **kw)
        ctx, ref = capi.Context(cfg), capi.Context(cfg)
        try:
            tops = torch.zeros(5, device="cuda")
            ctx.forward_async(x, labels, tops)               # returns 0
            ctx.backward_device_weight(torch.ones(1, device="cuda"), torch.empty_like(x))
            torch.cuda.synchronize()
            assert torch.isnan(tops).all(), tops
            with pytest.raises(capi.NpairError) as e:
                ctx.async_status()
            assert e.value.code == code
            ctx.async_status()                               # cleared
            if code == E_EMPTY_LIST:                         # then a synchronous step on good data
                _same(_sync_step(torch, ctx, x, l, 1.0), _sync_step(torch, ref, x, l, 1.0), "after the error")
        finally:
            ctx.close(); ref.close()


# ---------------------------------------------------------------------------------------------------------- 4. capture and replay
GRAPH_CASES = {
    "plain": dict(Q=512, D=128),
    "normalize_input": dict(Q=512, D=128, normalize_input=1, noise=3.0),
    "row blocks": dict(Q=900, D=128, sim_block_rows=256),
    "memory m=261": dict(Q=384, D=96, memory=(300, 261)),
    "no fused gradient": dict(Q=512, D=128, flags=capi.FLAG_NO_FUSED_GRAD),
}


class _Graphed:
    """A context, static input buffers and a CUDA graph of one asynchronous step over them."""

    def __init__(self, torch, cfg, M, x, l, mem):
        self.torch, self.ctx = torch, capi.Context(cfg, memory_rows=M)
        self.x, self.l = x.clone(), l.clone()
        self.mem = None if mem is None else (mem[0].clone(), mem[1].clone(), mem[2])
        self.lw = torch.ones(1, device="cuda")
        self.tops, self.dx = torch.zeros(5, device="cuda"), torch.zeros_like(x)
        _async_step(torch, self.ctx, self.x, self.l, 1.0, self.mem)      # warm-up: loads the kernels before the capture
        self.g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g):
            self.enqueue()

    def enqueue(self):
        if self.mem is None:
            self.ctx.forward_async(self.x, self.l, self.tops)
        else:
            self.ctx.forward_memory_async(self.x, self.l, *self.mem, self.tops)
        self.ctx.backward_device_weight(self.lw, self.dx)

    def replay(self, x, l, lw, mem=None):
        self.x.copy_(x); self.l.copy_(l); self.lw.fill_(lw)
        if mem is not None:
            self.mem[0].copy_(mem[0]); self.mem[1].copy_(mem[1])
        self.g.replay()
        self.torch.cuda.synchronize()
        return self.tops.cpu().numpy(), self.dx.cpu().numpy()


@pytest.mark.parametrize("name", list(GRAPH_CASES))
def test_capture_and_replay(torch, name):
    """Five batches replayed through the static buffers, each bit for bit a synchronous step on a separate context; then eager
    steps on the same context interleaved with replays, on the replay's stream and on another stream ordered explicitly."""
    cfg, M, x0, l0, mem0 = _case(torch, GRAPH_CASES[name], seed=40)
    G = _Graphed(torch, cfg, M, x0, l0, mem0)
    ref = capi.Context(cfg, memory_rows=M)
    try:
        batches = [_case(torch, GRAPH_CASES[name], seed=41 + b)[2:] for b in range(5)]
        lws = [1.0, 0.5, 1.3, 2.0 ** -20, -1.0]
        for b, (x, l, mem) in enumerate(batches):
            _same(G.replay(x, l, lws[b], mem), _sync_step(torch, ref, x, l, lws[b], mem), f"{name} replay {b}")
        # eager steps between replays, on the replay's stream
        for b, (x, l, mem) in enumerate(batches[:2]):
            _same(_sync_step(torch, G.ctx, x, l, 0.5, mem), _sync_step(torch, ref, x, l, 0.5, mem), f"{name} eager {b}")
            _same(G.replay(*batches[b + 2][:2], 1.0, batches[b + 2][2]), _sync_step(torch, ref, *batches[b + 2][:2], 1.0, batches[b + 2][2]),
                  f"{name} replay after eager {b}")
        # an eager step on another stream, ordered against the replays explicitly
        x, l, mem = batches[4]
        side, main = torch.cuda.Stream(), torch.cuda.current_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            got = _async_step(torch, G.ctx, x, l, 1.3, mem)
        main.wait_stream(side)
        _same(got, _sync_step(torch, ref, x, l, 1.3, mem), f"{name} eager on another stream")
        _same(G.replay(*batches[0][:2], 2.0, batches[0][2]), _sync_step(torch, ref, *batches[0][:2], 2.0, batches[0][2]),
              f"{name} replay after the other stream")
        G.ctx.async_status()
    finally:
        G.ctx.close(); ref.close()


# ---------------------------------------------------------------------------------------------------------- 5. refusals
def test_synchronous_calls_are_refused_during_a_capture(torch):
    Q, D = 256, 64
    cfg = capi.make_config(Q, D, **USAGE)
    x, l = _inputs(torch, Q, D, 50)
    ref, ctx, prof = capi.Context(cfg), capi.Context(cfg), capi.Context(cfg)
    tops, dx, lw = torch.zeros(5, device="cuda"), torch.zeros_like(x), torch.ones(1, device="cuda")
    host = (C.c_float * 5)()
    try:
        _async_step(torch, ctx, x, l, 1.0)
        _async_step(torch, prof, x, l, 1.0)
        prof.profile_enable(True)
        L = capi.lib()
        g = torch.cuda.CUDAGraph()
        codes = {}
        with torch.cuda.graph(g):
            st = torch.cuda.current_stream().cuda_stream
            ctx.forward_async(x, l, tops)
            n0 = capi.kernel_launches()
            codes["forward"] = L.npair_forward(ctx._h, x.data_ptr(), l.data_ptr(), host, st)
            codes["forward_memory"] = L.npair_forward_memory(ctx._h, x.data_ptr(), l.data_ptr(), None, None, 0, host, st)
            f = L.npair_forward_backward
            f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.POINTER(C.c_float), C.c_void_p]
            codes["forward_backward"] = f(ctx._h, x.data_ptr(), l.data_ptr(), 1.0, dx.data_ptr(), host, st)
            codes["forward_gathered"] = L.npair_forward_gathered(ctx._h, x.data_ptr(), l.data_ptr(), host, st)
            buf = np.zeros(Q, np.float32)
            codes["debug_read"] = L.npair_debug_read(ctx._h, 1, buf.ctypes.data_as(C.POINTER(C.c_float)), Q)
            ms = (C.c_float * 9)()
            codes["profile_read"] = L.npair_profile_read(ctx._h, ms)
            codes["async_status"] = L.npair_async_status(ctx._h)
            codes["profiled forward_async"] = L.npair_forward_async(prof._h, x.data_ptr(), l.data_ptr(), tops.data_ptr(), st)
            n1 = capi.kernel_launches()
            ctx.backward_device_weight(lw, dx)
        assert codes == {k: E_STATE for k in codes}, codes
        assert n1 == n0
        g.replay()
        torch.cuda.synchronize()
        _same((tops.cpu().numpy(), dx.cpu().numpy()), _sync_step(torch, ref, x, l, 1.0), "capture with refusals")
        ctx.debug_read(1, Q)                                 # after the capture the stream-less calls work again
        ctx.async_status()
    finally:
        ref.close(); ctx.close(); prof.close()


def test_world_2_refuses_the_asynchronous_calls(torch):
    Q, D = 64, 32
    ctx = capi.Context(capi.make_config(Q, D, world=2, rank=0))       # external collectives
    x, l = _inputs(torch, 2 * Q, D, 51)
    tops, dx, lw = torch.zeros(5, device="cuda"), torch.zeros(Q, D, device="cuda"), torch.ones(1, device="cuda")
    L, st = capi.lib(), torch.cuda.current_stream().cuda_stream
    try:
        ctx.forward_gathered(x, l)
        torch.cuda.synchronize()
        n0 = capi.kernel_launches()
        assert L.npair_forward_async(ctx._h, x.data_ptr(), l.data_ptr(), tops.data_ptr(), st) == E_ARG
        assert L.npair_forward_memory_async(ctx._h, x.data_ptr(), l.data_ptr(), None, None, 0, tops.data_ptr(), st) == E_ARG
        assert L.npair_backward_device_weight(ctx._h, lw.data_ptr(), dx.data_ptr(), st) == E_ARG
        assert L.npair_async_status(ctx._h) == E_ARG
        assert capi.kernel_launches() == n0
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------- 6. a whole torch step
def _trunk(torch, D_in, D):
    torch.manual_seed(1234)
    return torch.nn.Sequential(torch.nn.Linear(D_in, 256), torch.nn.ReLU(), torch.nn.Linear(256, D)).cuda()


def test_whole_torch_step_captured(torch):
    """Linear trunk -> NPairLoss(blocking=False) -> backward -> SGD captured with torch.cuda.graph, four batches replayed: the
    parameters equal, bit for bit, four eager steps with blocking=True."""
    Q, D_in, D = 256, 64, 512
    data = [_inputs(torch, Q, D_in, 60 + b, noise=0.5) for b in range(6)]
    net, net_ref = _trunk(torch, D_in, D), _trunk(torch, D_in, D)
    loss_fn, loss_ref = torch_api.NPairLoss(blocking=False, normalize_input=1, **USAGE), torch_api.NPairLoss(normalize_input=1, **USAGE)
    opt, opt_ref = torch.optim.SGD(net.parameters(), lr=0.5), torch.optim.SGD(net_ref.parameters(), lr=0.5)

    def step(n, f, o, x, l):
        o.zero_grad(set_to_none=True)
        loss, _ = f(n(x), l)
        loss.backward()
        o.step()
        return loss

    sx, sl = data[0][0].clone(), data[0][1].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                            # warm-up, two eager steps each
        for b in range(2):
            sx.copy_(data[b][0]); sl.copy_(data[b][1])
            step(net, loss_fn, opt, sx, sl)
    torch.cuda.current_stream().wait_stream(side)
    for b in range(2):
        step(net_ref, loss_ref, opt_ref, *data[b])
    g = torch.cuda.CUDAGraph()
    opt.zero_grad(set_to_none=True)
    with torch.cuda.graph(g):
        sloss, _ = loss_fn(net(sx), sl)
        sloss.backward()
        opt.step()
    for b in range(2, 6):
        sx.copy_(data[b][0]); sl.copy_(data[b][1])
        g.replay()
        lr = step(net_ref, loss_ref, opt_ref, *data[b])
        torch.cuda.synchronize()
        np.testing.assert_array_equal(_bits(sloss), _bits(lr), err_msg=f"loss of batch {b}")
    for (n, p), p_ref in zip(net.named_parameters(), net_ref.parameters()):
        np.testing.assert_array_equal(_bits(p), _bits(p_ref), err_msg=n)
    loss_fn.async_status()


def test_memory_ring_nonblocking_is_eager_only(torch):
    Q, D, M = 128, 64, 300
    loss_fn, loss_ref = torch_api.NPairLoss(memory_rows=M, blocking=False, **USAGE), torch_api.NPairLoss(memory_rows=M, **USAGE)
    for b in range(4):
        x, l = _inputs(torch, Q, D, 70 + b)
        xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        la, ta = loss_fn(xa, l)
        lb, tb = loss_ref(xb, l)
        la.backward(); lb.backward()
        np.testing.assert_array_equal(_bits(ta), _bits(tb), err_msg=f"tops of step {b}")
        np.testing.assert_array_equal(_bits(xa.grad), _bits(xb.grad), err_msg=f"gradient of step {b}")
    x, l = _inputs(torch, Q, D, 80)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="memory ring"):
        with torch.cuda.graph(g):
            loss_fn(x, l)
    loss_fn.async_status()
