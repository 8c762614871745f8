"""CPU-side checks of MAP@R evaluation (include/npair_b200.h, DESIGN 8): its symbols are exported, the device memory it adds is linear in
the number of positive pairs, it validates its arguments, and it fails loudly (no CPU fallback) when no device is present."""
import ctypes as C

import pytest

from npairloss_b200 import capi

MAP_SYMBOLS = ["npair_eval_map_at_r", "npair_eval_map_at_r_bytes"]


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_map_symbols_declared_and_exported():
    L = capi.lib()
    for s in MAP_SYMBOLS:
        assert s in capi.EXPORTS
        assert hasattr(L, s), s


def test_map_bytes_linear_in_positive_pairs():
    b = capi.eval_map_at_r_bytes
    for nq in (1, 1000, 60502):
        base = b(nq, 0)
        assert 12 * nq <= base <= 12 * nq + 64                       # per query: offset, gather counter
        for sum_r in (1, 7, 1 << 20, 60502 * 4, 3 * 196608, 1 << 33):
            assert b(nq, sum_r) - base == 8 * sum_r                 # value + histogram word per positive pair
    assert b(1000, 2 * 10**6) - b(1000, 10**6) == b(1000, 10**6) - b(1000, 0)


@pytest.mark.parametrize("nq,sum_r", [(0, 10), (-3, 10), (10, -1)])
def test_map_bytes_invalid(nq, sum_r):
    assert capi.eval_map_at_r_bytes(nq, sum_r) == 0


def test_map_call_without_evaluator():
    L = capi.lib()
    assert L.npair_eval_map_at_r(None, None, None, 1, None, None, 1, -1, None, None, None, None, None) == -1


def test_retrieval_metrics_rejects_cpu_tensors():
    torch = pytest.importorskip("torch")
    from npairloss_b200.torch_api import retrieval_metrics
    with pytest.raises(TypeError):
        retrieval_metrics(torch.zeros(8, 4), torch.zeros(8))


@pytest.mark.skipif(_have_gpu(), reason="checks the no-GPU failure mode")
def test_map_no_cpu_fallback():
    with pytest.raises(capi.NpairError) as e:
        capi.Evaluator(100, 200, 64).map_at_r(None, None, None, None)
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)
