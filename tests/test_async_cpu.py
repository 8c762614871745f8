"""The asynchronous step without a GPU (DESIGN 4.4): the C ABI's new symbols and their argument checks, and the autograd plumbing of
NPairLoss(blocking=False) with a stand-in context: the tops stay a device-side tensor, the loss weight reaches the library as a
one-element tensor instead of a host float, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from npairloss_b200 import capi, torch_api

ASYNC_SYMBOLS = ["npair_forward_async", "npair_forward_memory_async", "npair_backward_device_weight", "npair_async_status"]


def test_symbols_are_exported():
    L = capi.lib()
    for s in ASYNC_SYMBOLS:
        assert hasattr(L, s) and s in capi.EXPORTS, s


def test_null_context_is_an_argument_error():
    L = capi.lib()
    p = C.c_void_p(16)
    assert L.npair_forward_async(None, p, p, p, None) == -1
    assert L.npair_forward_memory_async(None, p, p, p, p, 1, p, None) == -1
    assert L.npair_backward_device_weight(None, p, p, None) == -1
    assert L.npair_async_status(None) == -1


class FakeContext:
    """Records what reaches the library; the tops and the gradient are made up."""

    def __init__(self, cfg, nccl_id, memory_rows=0):
        self.cfg, self.calls = cfg, []

    def forward_async(self, feat, label, tops_out):
        self.calls.append(("fwd_async", tuple(feat.shape), tuple(tops_out.shape)))
        tops_out.copy_(torch.tensor([1.25, 0.5, 0.75, 1.0, 3.0]))
        return tops_out

    def forward_memory_async(self, feat, label, mem_x, mem_l, m, tops_out):
        self.calls.append(("fwd_mem_async", int(m)))
        tops_out.copy_(torch.tensor([2.5, 0.0, 0.0, 0.0, 1.0]))
        return tops_out

    def backward_device_weight(self, loss_weight, diff):
        assert isinstance(loss_weight, torch.Tensor) and loss_weight.dtype == torch.float32 and loss_weight.numel() == 1
        self.calls.append(("bwd_dev", loss_weight.clone(), tuple(diff.shape)))
        diff.copy_(2.0 * loss_weight.expand_as(diff))

    def async_status(self):
        self.calls.append(("status",))


def _module(**kw):
    made = []

    def factory(cfg, nid):
        made.append(FakeContext(cfg, nid)); return made[-1]

    return torch_api.NPairLoss(_context_factory=factory, blocking=False, **kw), made


def test_nonblocking_plumbing():
    m, made = _module()
    x = torch.randn(6, 4, requires_grad=True)
    loss, tops = m(x, torch.tensor([0, 0, 1, 1, 2, 2]))
    assert loss.item() == 1.25 and tops.tolist() == [1.25, 0.5, 0.75, 1.0, 3.0] and not tops.requires_grad
    (3.0 * loss).backward()
    calls = made[0].calls
    assert calls[0] == ("fwd_async", (6, 4), (5,))
    assert calls[1][0] == "bwd_dev" and calls[1][1].tolist() == [3.0] and calls[1][2] == (6, 4)
    np.testing.assert_array_equal(x.grad.numpy(), np.full((6, 4), 6.0, np.float32))
    m.async_status()
    assert calls[-1] == ("status",)


def test_nonblocking_true_gradient_doubles_on_the_device():
    m, made = _module(true_gradient=True)
    x = torch.randn(4, 3, requires_grad=True)
    m(x, torch.tensor([0, 0, 1, 1]))[0].backward()
    np.testing.assert_array_equal(x.grad.numpy(), np.full((4, 3), 4.0, np.float32))


def test_nonblocking_memory_ring_runs_eagerly():
    made = []

    def factory(cfg, nid):
        made.append(FakeContext(cfg, nid, memory_rows=8)); return made[-1]

    m = torch_api.NPairLoss(_context_factory=factory, blocking=False, memory_rows=8)
    for step in range(3):
        loss, _ = m(torch.randn(4, 3), torch.tensor([0, 0, 1, 1]))
        assert loss.item() == 2.5
    assert [c[1] for c in made[0].calls if c[0] == "fwd_mem_async"] == [0, 4, 8]


def test_async_status_before_any_forward_is_a_no_op():
    m, made = _module()
    m.async_status()
    assert made == []


def test_nonblocking_needs_world_1():
    with pytest.raises(ValueError):
        torch_api.NPairLoss(world=2, blocking=False)
