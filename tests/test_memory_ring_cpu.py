"""NPairLoss(library_memory=True) plumbing with a stand-in context (no GPU): which entry each step takes, the ring carried into a context
re-created for a new batch size, the reset, memory() and the capture refusals; and the ring context's workspace against the memory
context's."""
import ctypes as C

import pytest
import torch

from npairloss_b200 import capi, torch_api


class FakeRingContext:
    """Keeps a ring as the library does: slot (count + i) mod M, a batch larger than M leaving its last M rows."""

    def __init__(self, cfg, nid, M):
        self.cfg, self.memory_rows, self.calls = cfg, M, []
        self.x, self.l, self.count = torch.zeros(M, cfg.D), torch.zeros(M), 0

    def _push(self, feat, label):
        q = feat.shape[0]
        for r in range(max(0, q - self.memory_rows), q):
            s = (self.count + r) % self.memory_rows
            self.x[s], self.l[s] = feat[r], label[r]
        self.count += q

    def forward_ring(self, feat, label):
        self.calls.append(("fwd_ring", min(self.count, self.memory_rows)))
        self._push(feat, label)
        return [1.5, 0.0, 0.0, 0.0, 0.0]

    def forward_ring_async(self, feat, label, tops):
        self.calls.append(("fwd_ring_async", min(self.count, self.memory_rows)))
        self._push(feat, label)
        tops.fill_(2.5)
        return tops

    def ring_read(self, rows, labels, count):
        self.calls.append(("read",))
        rows.copy_(self.x); labels.copy_(self.l); count.fill_(self.count)

    def ring_load(self, rows, labels, count):
        self.calls.append(("load", count))
        m = min(count, self.memory_rows)
        if m:
            self.x[:m], self.l[:m] = rows[:m], labels[:m]
        self.count = count

    def backward(self, lw, diff):
        diff.fill_(lw)

    def close(self):
        self.calls.append(("close",))


def _module(M=10, **kw):
    made = []

    def factory(cfg, nid):
        made.append(FakeRingContext(cfg, nid, M)); return made[-1]

    return torch_api.NPairLoss(_context_factory=factory, memory_rows=M, library_memory=True, **kw), made


def test_steps_go_through_the_ring_entries():
    m, made = _module()
    for step in range(3):
        loss, _ = m(torch.full((4, 3), float(step)), torch.tensor([0, 0, 1, 1]))
        assert loss.item() == 1.5
    assert made[0].calls == [("fwd_ring", 0), ("fwd_ring", 4), ("fwd_ring", 8)]
    m2, made2 = _module(blocking=False)
    loss, _ = m2(torch.ones(4, 3), torch.tensor([0, 0, 1, 1]))
    assert loss.item() == 2.5 and made2[0].calls == [("fwd_ring_async", 0)]


def test_new_batch_size_carries_the_ring_over():
    m, made = _module(M=10)
    for step in range(3):
        m(torch.full((4, 3), float(step)), torch.full((4,), float(step)))
    m(torch.full((6, 3), 7.0), torch.full((6,), 7.0))
    old, new = made
    assert old.calls[-2:] == [("read",), ("close",)]
    assert new.calls[0] == ("load", 12) and new.calls[1] == ("fwd_ring", 10)
    # slots as NPairLoss's own ring has them: 12 rows pushed, then 6 more from slot 2
    assert new.l.tolist() == [2.0, 2.0, 7.0, 7.0, 7.0, 7.0, 7.0, 7.0, 2.0, 2.0]
    rows, labels = m.memory()
    assert rows.shape == (10, 3) and labels.tolist() == new.l.tolist()
    # a new dimension starts an empty ring
    m(torch.ones(6, 5), torch.zeros(6))
    assert made[2].calls == [("fwd_ring", 0)]


def test_reset_and_memory():
    m, made = _module(M=10)
    assert m.memory() == (None, None)
    m(torch.ones(4, 3), torch.zeros(4))
    rows, labels = m.memory()
    assert rows.shape == (4, 3) and torch.equal(rows, torch.ones(4, 3))
    rows.zero_()                                        # a copy: the ring keeps its rows
    assert torch.equal(made[0].x[:4], torch.ones(4, 3))
    m.reset_memory()
    assert made[0].calls[-1] == ("load", 0)
    assert m.memory()[0].shape == (0, 3)
    m(torch.ones(4, 3), torch.zeros(4))
    assert made[0].calls[-1] == ("fwd_ring", 0)


def test_capture_refusals():
    m, _ = _module(M=10, blocking=False)
    x = torch.ones(4, 3)
    assert "eager step with this batch shape" in m._capture_refusal(x)
    m(x, torch.zeros(4))
    assert m._capture_refusal(x) == ("NPairLoss(library_memory=True) can be captured once its memory ring is full: 6 of its 10 rows are "
                                     "missing; run 2 more eager step(s) of 4 rows first")
    m(x, torch.zeros(4)); m(x, torch.zeros(4))
    assert m._capture_refusal(x) is None
    mb, _ = _module(M=10)
    mb(x, torch.zeros(4))
    assert "blocking=False" in mb._capture_refusal(x)
    with pytest.raises(ValueError, match="memory_rows"):
        torch_api.NPairLoss(library_memory=True)


@pytest.mark.parametrize("Q,M,D", [(200, 700, 101), (64, 256, 64), (256, 100, 32), (8, 0, 16)])
def test_ring_workspace(Q, M, D):
    """The ring's buffers on top of the memory context's: rows, labels, row maxima, two words per 32-row tile, the 32-byte state."""
    L = capi.lib()
    cfg = capi.make_config(Q, D)
    tiles = -(-(Q + M) // 32)
    extra = L.npair_memory_ring_workspace_bytes(C.byref(cfg), M) - L.npair_memory_workspace_bytes(C.byref(cfg), M)
    assert extra == 4 * M * D + 8 * M + 8 * tiles + 32


def test_ring_workspace_refuses_what_memory_refuses():
    L = capi.lib()
    for kw, M in ((dict(world=2), 5), (dict(gemm_backend=capi.GEMM_SIMT_CHECK), 5), (dict(global_scope=1), 5),
                  (dict(sim_block_rows=128), 5), ({}, -1)):
        cfg = capi.make_config(512, 32, **kw)
        assert L.npair_memory_ring_workspace_bytes(C.byref(cfg), M) == 0 == L.npair_memory_workspace_bytes(C.byref(cfg), M), kw
