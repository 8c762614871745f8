"""CPU-side checks of k-means evaluation (include/npair_b200.h, DESIGN 8.2): the NMI / F1 bookkeeping on known answers, the exported
symbols, the device-memory formula and its argument checks, and the loud failure (no CPU fallback) without a device."""
import math

import pytest

from npairloss_b200 import capi

KMEANS_SYMBOLS = ["npair_eval_kmeans", "npair_eval_kmeans_bytes"]


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def _scores(labels, assign):
    torch = pytest.importorskip("torch")
    from npairloss_b200.torch_api import clustering_scores
    return clustering_scores(torch.tensor(labels, dtype=torch.float32), torch.tensor(assign, dtype=torch.int32))


def test_perfect_clustering_scores_one():
    assert _scores([0, 0, 1, 1, 1, 2], [5, 5, 0, 0, 0, 9]) == (1.0, 1.0)
    assert _scores([2.5, 2.5, -1.0, -1.0], [1, 1, 0, 0]) == (1.0, 1.0)


def test_two_by_two_contingency():
    # labels a a a b b b, clusters 0 0 1 1 1 1: cells (a,0)=2 (a,1)=1 (b,1)=3, n_l = 3 3, n_c = 2 4
    nmi, f1 = _scores([0, 0, 0, 1, 1, 1], [0, 0, 1, 1, 1, 1])
    n = 6
    mi = 2 / n * math.log(n * 2 / (3 * 2)) + 1 / n * math.log(n * 1 / (3 * 4)) + 3 / n * math.log(n * 3 / (3 * 4))
    hy = math.log(2)
    hc = -(2 / n * math.log(2 / n) + 4 / n * math.log(4 / n))
    assert abs(nmi - 2 * mi / (hy + hc)) <= 1e-15
    tp, pc, pl = 1 + 0 + 3, 1 + 6, 3 + 3                           # C(2,2) + C(1,2) + C(3,2); C(2,2) + C(4,2); C(3,2) * 2
    p, r = tp / pc, tp / pl
    assert abs(f1 - 2 * p * r / (p + r)) <= 1e-15


def test_invariant_under_cluster_relabelling():
    lab = [0, 0, 1, 1, 2, 2, 2, 3, 1, 0]
    a = [0, 1, 1, 2, 2, 2, 3, 3, 0, 0]
    perm = {0: 7, 1: 3, 2: 0, 3: 11}
    nmi, f1 = _scores(lab, a)
    nmi2, f12 = _scores(lab, [perm[c] for c in a])
    assert abs(nmi - nmi2) <= 1e-15 and f1 == f12
    assert 0.0 < nmi < 1.0 and 0.0 < f1 < 1.0


def test_singleton_and_one_cluster_conventions():
    # every point its own cluster and its own label: NMI 1 (equal entropies), F1 0 (no pairs anywhere: 0/0 terms count as 0)
    assert _scores([0, 1, 2, 3], [3, 2, 1, 0]) == (1.0, 0.0)
    # one label, one cluster: both entropies 0, NMI 1; every pair agrees, F1 1
    assert _scores([4, 4, 4], [0, 0, 0]) == (1.0, 1.0)
    # one cluster over two labels: H(C) = 0 and I = 0, NMI 0; precision 2/6, recall 1
    nmi, f1 = _scores([0, 0, 1, 1], [0, 0, 0, 0])
    assert nmi == 0.0 and abs(f1 - 2 * (2 / 6) / (2 / 6 + 1)) <= 1e-15
    # singleton clusters over one label: precision 0/0 -> 0, recall 0 -> F1 0
    assert _scores([1, 1, 1], [0, 1, 2])[1] == 0.0


def test_kmeans_symbols_declared_and_exported():
    L = capi.lib()
    for s in KMEANS_SYMBOLS:
        assert s in capi.EXPORTS
        assert hasattr(L, s), s


def test_kmeans_bytes_formula():
    for n, k, D in ((1, 1, 1), (3000, 300, 200), (60502, 11316, 512), (5924, 100, 512)):
        assert capi.eval_kmeans_bytes(n, k, D) == 8 * k * D + 8 * n + 12 * k + 2064


@pytest.mark.parametrize("n,k,D", [(0, 1, 8), (10, 0, 8), (10, 11, 8), (10, 5, 0), (-1, -1, 4)])
def test_kmeans_bytes_invalid(n, k, D):
    assert capi.eval_kmeans_bytes(n, k, D) == 0


def test_kmeans_call_without_evaluator():
    L = capi.lib()
    assert L.npair_eval_kmeans(None, None, 1, 1, None, 1, None, None, None, None, None) == -1


def test_clustering_metrics_rejects_cpu_tensors():
    torch = pytest.importorskip("torch")
    from npairloss_b200.torch_api import clustering_metrics
    with pytest.raises(TypeError):
        clustering_metrics(torch.zeros(8, 4), torch.zeros(8))


@pytest.mark.skipif(_have_gpu(), reason="checks the no-GPU failure mode")
def test_kmeans_no_cpu_fallback():
    with pytest.raises(capi.NpairError) as e:
        capi.Evaluator(100, 10, 64)
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)
