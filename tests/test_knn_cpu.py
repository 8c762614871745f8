"""CPU-side checks of the k nearest neighbours (include/npair_b200.h, DESIGN 8.3): the exported symbols, the device-memory formula and
its argument checks, the call without an evaluator, and knn_merge's order (similarity descending, NaN last, then index) against numpy."""
import numpy as np
import pytest

from npairloss_b200 import capi

KNN_SYMBOLS = ["npair_eval_knn", "npair_eval_knn_bytes"]


def test_knn_symbols_declared_and_exported():
    L = capi.lib()
    for s in KNN_SYMBOLS:
        assert s in capi.EXPORTS
        assert hasattr(L, s), s


def test_knn_bytes_formula():
    for ng, k, br in ((1, 1, 128), (1003, 33, 256), (60502, 100, 1024), (12612, 1000, 4096), (20000, 1024, 128)):
        assert capi.eval_knn_bytes(ng, k, br) == 4 * br * ((ng + 31) // 32 * 32)
    assert capi.eval_knn_bytes(60502, 100, 0) == capi.eval_knn_bytes(60502, 100, 1024)


@pytest.mark.parametrize("ng,k,br", [(0, 1, 0), (10, 0, 0), (10, 11, 0), (2000, 1025, 0), (100, 5, 100), (100, 5, -128), (-1, -1, 0)])
def test_knn_bytes_invalid(ng, k, br):
    assert capi.eval_knn_bytes(ng, k, br) == 0


def test_knn_call_without_evaluator():
    import ctypes as C
    L = capi.lib()
    assert L.npair_eval_knn(None, None, 1, None, 1, -1, 0, C.c_float(-1.0), 1, 0, None, None, None) == -1


def test_knn_rejects_cpu_tensors():
    torch = pytest.importorskip("torch")
    from npairloss_b200.torch_api import knn
    with pytest.raises(TypeError):
        knn(torch.zeros(8, 4), k=2)


def test_knn_merge_order():
    """Three shard lists with ties across shards, -inf and NaN: the merge equals a numpy lexsort (NaN last, then s descending, then index)."""
    torch = pytest.importorskip("torch")
    from npairloss_b200.torch_api import knn_merge
    rng = np.random.default_rng(20261026)
    nq = 50
    sims, idxs = [], []
    for a, b, k in ((0, 40, 12), (40, 90, 12), (90, 200, 7)):
        s = rng.integers(-3, 4, size=(nq, k)).astype(np.float32) / 4     # few distinct values: ties across the shards
        s[rng.random((nq, k)) < 0.05] = -np.inf
        s[rng.random((nq, k)) < 0.05] = np.nan
        ix = np.stack([rng.choice(np.arange(a, b), size=k, replace=False) for _ in range(nq)]).astype(np.int32)
        sims.append(s)
        idxs.append(ix)
    s_all, i_all = np.concatenate(sims, 1), np.concatenate(idxs, 1).astype(np.int64)
    nan = np.isnan(s_all)
    order = np.lexsort((i_all, np.where(nan, 0.0, -s_all.astype(np.float64)), nan), axis=-1)
    for k in (1, 10, 31):
        ms, mi = knn_merge([torch.from_numpy(s) for s in sims], [torch.from_numpy(i) for i in idxs], k)
        assert mi.dtype == torch.int64 and ms.dtype == torch.float32
        want_i = np.take_along_axis(i_all, order[:, :k], 1)
        want_s = np.take_along_axis(s_all, order[:, :k], 1)
        np.testing.assert_array_equal(mi.numpy(), want_i)
        np.testing.assert_array_equal(ms.numpy(), want_s)       # NaN positions equal too
    with pytest.raises(ValueError):
        knn_merge([torch.from_numpy(s) for s in sims], [torch.from_numpy(i) for i in idxs], 32)
