"""CPU-side checks of hard negative class mining (include/npair_b200.h, DESIGN 8.4): the exported symbols, the device-memory formula and
its argument checks, the call without an evaluator, CPU tensors refused, the pools hard_class_batches draws, and class_embeddings
against the k-means fixed-point update of eval_ref bit for bit."""
import ctypes as C

import numpy as np
import pytest

from eval_ref import update_ref
from npairloss_b200 import capi

CLASS_BATCH_SYMBOLS = ["npair_eval_class_batches", "npair_eval_class_batches_bytes"]


def test_class_batch_symbols_declared_and_exported():
    L = capi.lib()
    for s in CLASS_BATCH_SYMBOLS:
        assert s in capi.EXPORTS
        assert hasattr(L, s), s


def test_class_batches_bytes_formula():
    for C_, P, b in ((2, 2, 1), (1003, 77, 5), (11318, 11318, 189), (40000, 16384, 132), (16384, 16384, 1)):
        assert capi.eval_class_batches_bytes(C_, P, b) == 4 * C_ * ((C_ + 31) // 32 * 32) + 4 * b * P
    assert capi.eval_class_batches_bytes(11318, 11318, 189) < 522e6      # SOP-sized


@pytest.mark.parametrize("C_,P,b", [(0, 2, 1), (10, 1, 1), (10, 11, 1), (20000, 16385, 1), (10, 5, 0), (-1, -1, -1)])
def test_class_batches_bytes_invalid(C_, P, b):
    assert capi.eval_class_batches_bytes(C_, P, b) == 0


def test_class_batches_call_without_evaluator():
    pools = (C.c_int32 * 4)(0, 1, 1, 0)
    assert capi.lib().npair_eval_class_batches(None, None, 2, pools, 2, 2, 2, None, None, None) == -1


def test_class_batches_rejects_cpu_tensors():
    torch = pytest.importorskip("torch")
    from npairloss_b200.torch_api import class_embeddings, hard_class_batches
    with pytest.raises(TypeError):
        hard_class_batches(torch.zeros(8, 4), 2, 1)
    with pytest.raises(TypeError):
        hard_class_batches(torch.zeros(8, 4, dtype=torch.float64), 2, 1)
    with pytest.raises(TypeError):
        class_embeddings(torch.zeros(8, 4), torch.zeros(8))               # normalize=True runs on the GPU only
    with pytest.raises(TypeError):
        class_embeddings(torch.zeros(8, 4, dtype=torch.float64), torch.zeros(8), normalize=False)


def test_hard_class_batches_pools(monkeypatch):
    """The pools are torch.randperm(C, generator=g)[:P] for t = 0, 1, ... with g seeded by `seed`, P = min(C, 16384) by default, handed
    to the evaluator in that order; the same seed gives the same pools."""
    torch = pytest.importorskip("torch")
    from npairloss_b200 import torch_api

    seen = []

    class FakeEvaluator:
        def __init__(self, *a):
            self.args = a

        def class_batches(self, x, pools, n):
            seen.append((self.args, np.asarray(pools).copy(), n))
            b = np.asarray(pools).shape[0]
            return torch.zeros(b, n, dtype=torch.int32), torch.zeros(b, n)

        def close(self):
            pass

    monkeypatch.setattr(torch_api.capi, "Evaluator", FakeEvaluator)
    monkeypatch.setattr(torch_api, "_embeddings", lambda who, x: x)      # the fake takes CPU rows
    for C_, P, seed in ((50, None, 0), (50, 7, 3), (20000, None, 11)):
        x = torch.zeros(C_, 4)
        for _ in range(2):
            batches, _ = torch_api.hard_class_batches(x, 5, 6, pool_size=P, seed=seed)
            assert batches.dtype == torch.int64 and tuple(batches.shape) == (6, 5)
        g = torch.Generator().manual_seed(seed)
        want = np.stack([torch.randperm(C_, generator=g)[:min(C_, 16384) if P is None else P].numpy() for _ in range(6)])
        for args, pools, n in seen:
            np.testing.assert_array_equal(pools, want)
            assert n == 5 and args[:3] == (C_, C_, 4)
        seen.clear()


def test_class_embeddings_fixed_point_mean():
    """class_embeddings(normalize=False) equals eval_ref.update_ref bit for bit, classes in ascending label order, whatever the order of
    the examples and the label dtype; NaN labels raise."""
    torch = pytest.importorskip("torch")
    from npairloss_b200.torch_api import class_embeddings
    rng = np.random.default_rng(20261027)
    for n, D, scale in ((500, 37, 3.0), (2000, 128, 1e-3), (64, 8, 1.0)):
        x = (rng.standard_normal((n, D)) * scale).astype(np.float32)
        ids = np.array([-5.0, 2.0, 7.5, 100.0, 3.0, 0.0], np.float32)
        lab = ids[rng.integers(0, ids.size, size=n)]
        u = np.unique(lab)
        ref = update_ref(x, np.searchsorted(u, lab), np.zeros((u.size, D), np.float32))
        cl, ce = class_embeddings(torch.from_numpy(x), torch.from_numpy(lab), normalize=False)
        np.testing.assert_array_equal(cl.numpy(), u)
        np.testing.assert_array_equal(ce.numpy().view(np.uint32), ref.view(np.uint32))
        perm = rng.permutation(n)
        _, ce2 = class_embeddings(torch.from_numpy(x[perm]), torch.from_numpy(lab[perm].astype(np.float64)), normalize=False)
        np.testing.assert_array_equal(ce2.numpy().view(np.uint32), ref.view(np.uint32))
    lab = lab.copy()
    lab[3] = np.nan
    with pytest.raises(ValueError):
        class_embeddings(torch.from_numpy(x), torch.from_numpy(lab), normalize=False)
