"""Every forward and backward entry point of the C ABI refuses each precondition it checks, in a fixed order, before it enqueues anything.

For each refusal the test checks the return code and the start of the message, that no kernel was launched, and that the step the
context holds is the one it held before: the backward that follows gives, bit for bit, what it gives without the refused call.  Pairs of
conditions pin the order of the checks: null pointers, then a memory call's m and context, then the gradient's alignment, then the
step's own checks (no forward, the wrong backward mode, no communicator, a capturing stream, an asynchronous call at world > 1 or under
profiling in a capture).  The Python binding refuses a CPU, fp64, non-contiguous or too short tensor before any library call."""
import contextlib
import ctypes as C

import numpy as np
import pytest

from npairloss_b200 import capi, synth

pytestmark = pytest.mark.gpu

Q, D, M = 200, 72, 261
E_ARG, E_STATE = -1, -6
LW = 0.8


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need an H100"
    assert torch.cuda.get_device_capability(0) == (9, 0)
    return torch


def _bits(t):
    return np.ascontiguousarray(t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t, np.float32)).view(np.uint32)


@pytest.fixture(scope="module")
def data(torch):
    x, lab = synth.make_inputs(2 * Q + M, D, seed=77, imgs_per_class=4, noise=2.5)
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    return dict(x=xt[:Q].contiguous(), l=lt[:Q].contiguous(), xw=xt[:2 * Q].contiguous(), lw=lt[:2 * Q].contiguous(),
                xm=xt[2 * Q:].contiguous(), lm=lt[2 * Q:].contiguous())


# the contexts: "one" a world-1 context, "mem" a memory context of M rows, "rows" / "split" rank 0 of an emulated world of two without
# a communicator, in the row-record and the reduce-scatter backward mode
def _context(kind):
    if kind == "mem":
        return capi.Context(capi.make_config(Q, D, **synth.USAGE_MINING), memory_rows=M)
    if kind == "one":
        return capi.Context(capi.make_config(Q, D, **synth.USAGE_MINING))
    return capi.Context(capi.make_config(Q, D, world=2, rank=0, bwd_exchange=0 if kind == "rows" else 1, **synth.USAGE_MINING))


def _forward(ctx, kind, d):
    if kind == "mem":
        return ctx.forward_memory(d["x"], d["l"], d["xm"], d["lm"], M)
    if kind == "one":
        return ctx.forward(d["x"], d["l"])
    return ctx.forward_gathered(d["xw"], d["lw"])


def _backward(torch, ctx, kind):
    """The step's backward, its outputs as bits: the row records and the gradient, or both halves of the partial backward."""
    g = torch.full((Q, D), float("nan"), dtype=torch.float32, device="cuda")
    if kind == "rows":
        rec = torch.empty((Q, 8), dtype=torch.float32, device="cuda")
        ctx.row_scalars(rec)
        ctx.backward_gathered(LW, torch.cat([rec, rec]).contiguous(), g)
        out = [rec, g]
    elif kind == "split":
        th = torch.full((2 * Q, D), float("nan"), dtype=torch.float32, device="cuda")
        ctx.backward_partial(LW, g, th)
        out = [g, th]
    else:
        ctx.backward(LW, g)
        out = [g]
    torch.cuda.synchronize()
    return [_bits(t) for t in out]


@pytest.fixture(scope="module")
def reference(torch, data):
    ref = {}
    for kind in ("one", "mem", "rows", "split"):
        ctx = _context(kind)
        try:
            tops = _forward(ctx, kind, data)
            ref[kind] = (_bits(tops), _backward(torch, ctx, kind))
        finally:
            ctx.close()
    assert ref["one"][1][0].size and not np.isnan(ref["one"][1][0].view(np.float32)).any()
    return ref


@contextlib.contextmanager
def _capturing(torch):
    """A stream in a CUDA graph capture (with one node of its own, so the graph is not empty)."""
    s, g = torch.cuda.Stream(), torch.cuda.CUDAGraph()
    pad = torch.zeros(4, device="cuda")
    with torch.cuda.graph(g, stream=s):
        pad.add_(1.0)
        yield s.cuda_stream


class Args:
    """Pointers of the calls: valid device buffers, a gradient 4 bytes off the 16-byte grid, a host tops buffer."""

    def __init__(self, torch, d):
        self.x, self.l, self.xw, self.lw = (d[k].data_ptr() for k in ("x", "l", "xw", "lw"))
        self.xm, self.lm = d["xm"].data_ptr(), d["lm"].data_ptr()
        self.buf = torch.zeros(2 * Q * D + 8, dtype=torch.float32, device="cuda")
        self.rs = torch.zeros(2 * Q * 8, dtype=torch.float32, device="cuda")
        self.dtops = torch.zeros(8, dtype=torch.float32, device="cuda")
        self.wgt = torch.ones(1, dtype=torch.float32, device="cuda")
        self.g = self.buf.data_ptr()
        self.mis = self.g + 4
        self.host = (C.c_float * 5)()


# The refused calls: (id, context kind, forward first, stream kind, call, code, message start).  A call is f(L, h, a, st); stream kind
# "cap" runs it on a capturing stream, "prof" on a capturing stream with profiling on.
def _f(L, h, a, st, x=True, lab=True):
    return L.npair_forward(h, a.x if x else None, a.l if lab else None, a.host, st)


CASES = [
    # null pointers, alone and before a capturing stream, no communicator or a misaligned gradient
    ("forward/null", "one", True, None, lambda L, h, a, st: _f(L, h, a, st, lab=False), E_ARG, "null pointer"),
    ("forward/null+capture", "one", True, "cap", lambda L, h, a, st: _f(L, h, a, st, x=False), E_ARG, "null pointer"),
    ("forward/null+no-comm", "rows", True, None, lambda L, h, a, st: _f(L, h, a, st, x=False), E_ARG, "null pointer"),
    ("forward_async/null", "one", True, None, lambda L, h, a, st: L.npair_forward_async(h, a.x, None, a.dtops.data_ptr(), st), E_ARG,
     "null pointer"),
    ("forward_async/null+world2", "rows", True, None, lambda L, h, a, st: L.npair_forward_async(h, a.x, a.l, None, st), E_ARG,
     "null pointer"),
    ("forward_gathered/null", "rows", True, None, lambda L, h, a, st: L.npair_forward_gathered(h, a.xw, None, a.host, st), E_ARG,
     "null pointer"),
    ("forward_gathered/null+capture", "one", True, "cap", lambda L, h, a, st: L.npair_forward_gathered(h, None, a.l, a.host, st), E_ARG,
     "null pointer"),
    ("forward_memory/null", "mem", True, None, lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, None, a.lm, M, a.host, st), E_ARG,
     "null pointer"),
    ("forward_memory/null+m", "mem", True, None, lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, a.xm, None, M + 1, a.host, st),
     E_ARG, "null pointer"),
    ("forward_memory_async/null", "mem", True, None,
     lambda L, h, a, st: L.npair_forward_memory_async(h, a.x, a.l, a.xm, a.lm, M, None, st), E_ARG, "null pointer"),
    ("forward_backward/null", "one", True, None, lambda L, h, a, st: L.npair_forward_backward(h, a.x, a.l, LW, None, a.host, st), E_ARG,
     "null pointer"),
    ("forward_backward/null+misaligned", "one", True, None,
     lambda L, h, a, st: L.npair_forward_backward(h, None, a.l, LW, a.mis, a.host, st), E_ARG, "null pointer"),
    ("backward/null", "one", True, None, lambda L, h, a, st: L.npair_backward(h, LW, None, st), E_ARG, "null gradient"),
    ("backward/null+no-forward", "one", False, None, lambda L, h, a, st: L.npair_backward(h, LW, None, st), E_ARG, "null gradient"),
    ("backward_device_weight/null", "one", True, None, lambda L, h, a, st: L.npair_backward_device_weight(h, None, a.g, st), E_ARG,
     "null pointer"),
    ("backward_device_weight/null+world2", "rows", True, None, lambda L, h, a, st: L.npair_backward_device_weight(h, a.wgt.data_ptr(), None, st),
     E_ARG, "null pointer"),
    ("backward_partial/null", "split", True, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, a.g, None, st), E_ARG,
     "null gradient"),
    ("backward_partial/null+mode", "rows", True, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, None, a.g, st), E_ARG,
     "null gradient"),
    ("backward_gathered/null", "rows", True, None, lambda L, h, a, st: L.npair_backward_gathered(h, LW, None, a.g, st), E_ARG,
     "null pointer"),
    ("backward_gathered/null+no-forward", "rows", False, None, lambda L, h, a, st: L.npair_backward_gathered(h, LW, a.rs.data_ptr(), None, st),
     E_ARG, "null pointer"),
    # a memory call's m and context, before the alignment, the communicator and the capture checks
    ("forward_memory/m<0", "mem", True, None, lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, a.xm, a.lm, -1, a.host, st), E_ARG,
     "m = -1 memory rows outside [0, 261]"),
    ("forward_memory/m>M", "mem", True, None, lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, a.xm, a.lm, M + 1, a.host, st),
     E_ARG, "m = 262 memory rows outside [0, 261]"),
    ("forward_memory/m>M+capture", "mem", True, "cap",
     lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, a.xm, a.lm, M + 1, a.host, st), E_ARG, "m = 262"),
    ("forward_memory/m>0-plain", "one", True, None, lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, a.xm, a.lm, 1, a.host, st),
     E_ARG, "m = 1 memory rows outside [0, 0]"),
    ("forward_memory/world2", "rows", True, None, lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, None, None, 0, a.host, st),
     E_ARG, "a cross-batch memory needs world = 1"),
    ("forward_memory_async/m<0", "mem", True, None,
     lambda L, h, a, st: L.npair_forward_memory_async(h, a.x, a.l, a.xm, a.lm, -1, a.dtops.data_ptr(), st), E_ARG, "m = -1"),
    ("forward_memory_async/m>M+prof", "mem", True, "prof",
     lambda L, h, a, st: L.npair_forward_memory_async(h, a.x, a.l, a.xm, a.lm, M + 1, a.dtops.data_ptr(), st), E_ARG, "m = 262"),
    ("forward_memory_async/world2", "rows", True, None,
     lambda L, h, a, st: L.npair_forward_memory_async(h, a.x, a.l, a.xm, a.lm, 1, a.dtops.data_ptr(), st), E_ARG,
     "a cross-batch memory needs world = 1"),
    # a misaligned gradient, before the step's checks
    ("forward_backward/misaligned", "one", True, None, lambda L, h, a, st: L.npair_forward_backward(h, a.x, a.l, LW, a.mis, a.host, st),
     E_ARG, "the gradient pointer is not 16-byte aligned"),
    ("forward_backward/misaligned+capture", "one", True, "cap",
     lambda L, h, a, st: L.npair_forward_backward(h, a.x, a.l, LW, a.mis, a.host, st), E_ARG, "the gradient pointer is not"),
    ("forward_backward/misaligned+no-comm", "rows", True, None,
     lambda L, h, a, st: L.npair_forward_backward(h, a.x, a.l, LW, a.mis, a.host, st), E_ARG, "the gradient pointer is not"),
    ("backward/misaligned", "one", True, None, lambda L, h, a, st: L.npair_backward(h, LW, a.mis, st), E_ARG, "the gradient pointer is not"),
    ("backward/misaligned+no-forward", "one", False, None, lambda L, h, a, st: L.npair_backward(h, LW, a.mis, st), E_ARG,
     "the gradient pointer is not"),
    ("backward/misaligned+no-comm", "rows", True, None, lambda L, h, a, st: L.npair_backward(h, LW, a.mis, st), E_ARG,
     "the gradient pointer is not"),
    ("backward_device_weight/misaligned", "one", True, None,
     lambda L, h, a, st: L.npair_backward_device_weight(h, a.wgt.data_ptr(), a.mis, st), E_ARG, "the gradient pointer is not"),
    ("backward_device_weight/misaligned+no-forward", "one", False, None,
     lambda L, h, a, st: L.npair_backward_device_weight(h, a.wgt.data_ptr(), a.mis, st), E_ARG, "the gradient pointer is not"),
    ("backward_partial/misaligned-local", "split", True, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, a.mis, a.g, st), E_ARG,
     "d_local_half is not"),
    ("backward_partial/misaligned-total", "split", True, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, a.g, a.mis, st), E_ARG,
     "d_total_half is not"),
    ("backward_partial/misaligned+no-forward", "one", False, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, a.mis, None, st),
     E_ARG, "d_local_half is not"),
    ("backward_partial/misaligned+mode", "rows", True, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, a.g, a.mis, st), E_ARG,
     "d_total_half is not"),
    ("backward_gathered/misaligned", "rows", True, None,
     lambda L, h, a, st: L.npair_backward_gathered(h, LW, a.rs.data_ptr(), a.mis, st), E_ARG, "the gradient pointer is not"),
    ("backward_gathered/misaligned+mode+no-forward", "one", False, None,
     lambda L, h, a, st: L.npair_backward_gathered(h, LW, a.rs.data_ptr(), a.mis, st), E_ARG, "the gradient pointer is not"),
    # no forward yet, before the backward mode and the communicator
    ("backward/no-forward", "one", False, None, lambda L, h, a, st: L.npair_backward(h, LW, a.g, st), E_STATE,
     "npair_backward called without a successful forward"),
    ("backward/no-forward+no-comm", "rows", False, None, lambda L, h, a, st: L.npair_backward(h, LW, a.g, st), E_STATE,
     "npair_backward called without"),
    ("backward_device_weight/no-forward", "one", False, None,
     lambda L, h, a, st: L.npair_backward_device_weight(h, a.wgt.data_ptr(), a.g, st), E_STATE, "npair_backward_device_weight called without"),
    ("backward_partial/no-forward", "split", False, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, a.g, a.g, st), E_STATE,
     "npair_backward_partial called without"),
    ("backward_partial/no-forward+mode", "rows", False, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, a.g, a.g, st), E_STATE,
     "npair_backward_partial called without"),
    ("backward_gathered/no-forward+mode", "one", False, None,
     lambda L, h, a, st: L.npair_backward_gathered(h, LW, a.rs.data_ptr(), a.g, st), E_STATE, "npair_backward_gathered called without"),
    # the backward mode
    ("backward_partial/mode", "rows", True, None, lambda L, h, a, st: L.npair_backward_partial(h, LW, a.g, a.g, st), E_STATE,
     "this context exchanges row scalars"),
    ("backward_gathered/mode", "split", True, None, lambda L, h, a, st: L.npair_backward_gathered(h, LW, a.rs.data_ptr(), a.g, st), E_STATE,
     "this context does not exchange row scalars"),
    ("backward_gathered/mode-world1", "one", True, None, lambda L, h, a, st: L.npair_backward_gathered(h, LW, a.rs.data_ptr(), a.g, st),
     E_STATE, "this context does not exchange row scalars"),
    # no communicator, before a capturing stream
    ("forward/no-comm", "rows", True, None, lambda L, h, a, st: _f(L, h, a, st), E_STATE,
     "context was created without a communicator: use npair_forward_gathered"),
    ("forward/no-comm+capture", "split", True, "cap", lambda L, h, a, st: _f(L, h, a, st), E_STATE, "context was created without"),
    ("forward_backward/no-comm", "rows", True, None, lambda L, h, a, st: L.npair_forward_backward(h, a.x, a.l, LW, a.g, a.host, st),
     E_STATE, "context was created without a communicator: use npair_forward_gathered"),
    ("backward/no-comm", "rows", True, None, lambda L, h, a, st: L.npair_backward(h, LW, a.g, st), E_STATE,
     "context was created without a communicator: use npair_backward_partial / npair_backward_gathered"),
    # a synchronous call on a capturing stream
    ("forward/capture", "one", True, "cap", lambda L, h, a, st: _f(L, h, a, st), E_STATE, "npair_forward waits on the host"),
    ("forward_gathered/capture", "rows", True, "cap", lambda L, h, a, st: L.npair_forward_gathered(h, a.xw, a.lw, a.host, st), E_STATE,
     "npair_forward_gathered waits on the host"),
    ("forward_memory/capture", "mem", True, "cap", lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, a.xm, a.lm, M, a.host, st),
     E_STATE, "npair_forward_memory waits on the host"),
    ("forward_memory/m=0+capture", "mem", True, "cap", lambda L, h, a, st: L.npair_forward_memory(h, a.x, a.l, None, None, 0, a.host, st),
     E_STATE, "npair_forward waits on the host"),
    ("forward_backward/capture", "one", True, "cap", lambda L, h, a, st: L.npair_forward_backward(h, a.x, a.l, LW, a.g, a.host, st),
     E_STATE, "npair_forward_backward waits on the host"),
    # an asynchronous call at world 2, before profiling in a capture
    ("forward_async/world2", "rows", True, None, lambda L, h, a, st: L.npair_forward_async(h, a.x, a.l, a.dtops.data_ptr(), st), E_ARG,
     "npair_forward_async is world-1 only"),
    ("forward_async/world2+prof", "split", True, "prof", lambda L, h, a, st: L.npair_forward_async(h, a.x, a.l, a.dtops.data_ptr(), st),
     E_ARG, "npair_forward_async is world-1 only"),
    ("backward_device_weight/world2", "rows", True, None,
     lambda L, h, a, st: L.npair_backward_device_weight(h, a.wgt.data_ptr(), a.g, st), E_ARG, "npair_backward_device_weight is world-1 only"),
    ("backward_device_weight/world2+misaligned+no-forward", "split", False, None,
     lambda L, h, a, st: L.npair_backward_device_weight(h, a.wgt.data_ptr(), a.mis, st), E_ARG, "npair_backward_device_weight is world-1"),
    # an asynchronous call under profiling on a capturing stream, before the alignment and the forward
    ("forward_async/prof", "one", True, "prof", lambda L, h, a, st: L.npair_forward_async(h, a.x, a.l, a.dtops.data_ptr(), st), E_STATE,
     "npair_forward_async: profiling"),
    ("forward_memory_async/prof", "mem", True, "prof",
     lambda L, h, a, st: L.npair_forward_memory_async(h, a.x, a.l, a.xm, a.lm, M, a.dtops.data_ptr(), st), E_STATE,
     "npair_forward_memory_async: profiling"),
    ("forward_memory_async/m=0+prof", "mem", True, "prof",
     lambda L, h, a, st: L.npair_forward_memory_async(h, a.x, a.l, None, None, 0, a.dtops.data_ptr(), st), E_STATE,
     "npair_forward_async: profiling"),
    ("backward_device_weight/prof", "one", True, "prof",
     lambda L, h, a, st: L.npair_backward_device_weight(h, a.wgt.data_ptr(), a.g, st), E_STATE, "npair_backward_device_weight: profiling"),
    ("backward_device_weight/prof+misaligned+no-forward", "one", False, "prof",
     lambda L, h, a, st: L.npair_backward_device_weight(h, a.wgt.data_ptr(), a.mis, st), E_STATE, "npair_backward_device_weight: profiling"),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_refused_call_keeps_the_step(torch, data, reference, case):
    name, kind, forward_first, stream, call, code, msg = case
    L, a = capi.lib(), Args(torch, data)
    ctx = _context(kind)
    try:
        if forward_first:
            _forward(ctx, kind, data)
        if stream == "prof":
            ctx.profile_enable(True)
        torch.cuda.synchronize()
        launches = capi.kernel_launches()
        with _capturing(torch) if stream else contextlib.nullcontext(torch.cuda.current_stream().cuda_stream) as st:
            rc = call(L, ctx._h, a, st)
        err = L.npair_last_error(ctx._h).decode()
        assert capi.kernel_launches() == launches, f"{name}: a refused call launched kernels"
        assert rc == code, f"{name}: {rc} ({err})"
        assert err.startswith(msg), f"{name}: {err!r}"
        if stream == "prof":
            ctx.profile_enable(False)
        tops = _forward(ctx, kind, data) if not forward_first else None
        want_tops, want = reference[kind]
        if tops is not None:
            assert np.array_equal(_bits(tops), want_tops), name
        got = _backward(torch, ctx, kind)
        assert all(np.array_equal(g, w) for g, w in zip(got, want)), f"{name}: the backward after the refused call"
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------- the Python binding
def _bad_tensors(torch, t, short=True):
    """For a tensor t a call takes: a CPU copy, an fp64 copy, a non-contiguous view of its shape, and (short) a tensor one float too
    short, of 2-D rows one float too short."""
    out = [(t.cpu(), TypeError), (t.double(), TypeError)]
    if t.dim() == 2:
        out.append((torch.empty((t.shape[1], t.shape[0]), dtype=torch.float32, device="cuda").t(), TypeError))
    elif t.numel() > 1:
        out.append((torch.empty(2 * t.numel(), dtype=torch.float32, device="cuda")[::2].view(t.shape), TypeError))
    if short and t.numel() > 1:
        out.append((t[:, :-1].contiguous() if t.dim() == 2 else t.reshape(-1)[:-1].clone(), ValueError))
    return out


def _method_cases(torch, d):
    g = torch.zeros((Q, D), dtype=torch.float32, device="cuda")
    gw = torch.zeros((2 * Q, D), dtype=torch.float32, device="cuda")
    tops = torch.zeros(5, dtype=torch.float32, device="cuda")
    rec, rs = torch.zeros((Q, 8), device="cuda"), torch.zeros((2, Q, 8), device="cuda")
    w = torch.ones(1, dtype=torch.float32, device="cuda")
    x, lab, xw, lw, xm, lm = d["x"], d["l"], d["xw"], d["lw"], d["xm"], d["lm"]
    return [  # (context kind, method, arguments)
        ("one", "forward", [x, lab]),
        ("one", "forward_backward", [x, lab, LW, g]),
        ("one", "backward", [LW, g]),
        ("one", "forward_async", [x, lab, tops]),
        ("one", "backward_device_weight", [w, g]),
        ("one", "set_anchor_io", [lab, lab]),
        ("mem", "forward_memory", [x, lab, xm, lm, M]),
        ("mem", "forward_memory_async", [x, lab, xm, lm, M, tops]),
        ("rows", "forward_gathered", [xw, lw]),
        ("rows", "row_scalars", [rec]),
        ("rows", "backward_gathered", [LW, rs, g]),
        ("split", "backward_partial", [LW, g, gw]),
    ]


def test_context_methods_refuse_bad_tensors(torch, data):
    for kind, method, args in _method_cases(torch, data):
        ctx = _context(kind)
        try:
            _forward(ctx, kind, data)
            torch.cuda.synchronize()
            for i, good in enumerate(args):
                if not isinstance(good, torch.Tensor):
                    continue
                for bad, exc in _bad_tensors(torch, good):
                    launches = capi.kernel_launches()
                    with pytest.raises(exc):
                        getattr(ctx, method)(*args[:i], bad, *args[i + 1:])
                    assert capi.kernel_launches() == launches, (method, i)
        finally:
            ctx.close()


def test_evaluator_and_module_functions_refuse_bad_tensors(torch, data):
    x, lab = data["x"], data["l"]
    y, inv = capi.l2normalize_forward(x)
    cut = torch.zeros(Q, dtype=torch.float32, device="cuda")
    ev = capi.Evaluator(Q, Q, D)
    try:
        calls = [
            (ev.rank, [x, lab, x, lab]), (ev.best_positive, [x, lab, x, lab, 1.0]), (ev.count, [x, x, cut, 1.0]),
            (ev.knn, [x, x, 3]), (ev.map_at_r, [x, lab, x, lab]), (ev.kmeans, [x, 4, [0, 1, 2, 3], 2]), (ev.kmeans_seed, [x, 4, 1]),
            (ev.class_batches, [x, np.array([[0, 1, 2]], np.int32), 2]),
            (capi.l2normalize_forward, [x]), (capi.l2normalize_backward, [y, inv, x]),
            (capi.debug_gemm, [capi.PREC_FP32_FP16X2, capi.GEMM_TCGEN05, x, x]),
        ]
        shaping = {(capi.l2normalize_forward, 0), (capi.l2normalize_backward, 0), (capi.debug_gemm, 2)}   # these set the shape
        torch.cuda.synchronize()
        for fn, args in calls:
            for i, good in enumerate(args):
                if not isinstance(good, torch.Tensor):
                    continue
                for bad, exc in _bad_tensors(torch, good, short=(fn, i) not in shaping):
                    launches = capi.kernel_launches()
                    with pytest.raises(exc):
                        fn(*args[:i], bad, *args[i + 1:])
                    assert capi.kernel_launches() == launches, (fn.__name__, i)
    finally:
        ev.close()
