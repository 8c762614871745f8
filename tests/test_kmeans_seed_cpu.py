"""The k-means++ seeding rule's host reference (tests/kmeans_seed_ref.py, DESIGN 8.2): SplitMix64's known answers, the vectorised
reference against per-element loops, the first draw's frequencies, ties between trials, the phi = 0 fallback and the prefix property."""
import numpy as np
import pytest

import kmeans_seed_ref as R


def test_splitmix64_known_answers():
    assert [R.u(0, 0, j) for j in range(3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    assert R.u(0, 1, 0) == R.splitmix_mix((257 * R.GAMMA) & R.M64)          # number t * 256 + j + 1


def test_default_trials():
    assert [R.default_trials(k) for k in (1, 2, 3, 7, 8, 11316)] == [2, 2, 3, 3, 4, 11]


@pytest.mark.parametrize("n,D,k,L", [(1, 1, 1, 0), (2, 3, 2, 1), (9, 3, 5, 2), (31, 4, 10, 0), (40, 7, 40, 3)])
def test_reference_matches_brute_force(n, D, k, L):
    rng = np.random.default_rng(1000 + n)
    x = rng.standard_normal((n, D)).astype(np.float32)
    for seed in (0, 7, 2 ** 64 - 1):
        assert R.seed_rows(x, k, seed, L) == R.seed_rows_brute(x, k, seed, L)


def test_quantise_rounds_half_to_even_and_bounds():
    x = np.array([[0.75, -0.75, 3.0 / 16384, 5.0 / 16384, 0.0]], np.float32)   # sigma = 1: q = rint(x * 8192)
    np.testing.assert_array_equal(R.quantise(x), [[6144, -6144, 2, 2, 0]])
    y = np.array([[1.0, -1.0]], np.float32)                                     # sigma = 1/2: |q| = 2^12
    np.testing.assert_array_equal(R.quantise(y), [[4096, -4096]])
    assert np.abs(R.quantise(np.random.default_rng(0).standard_normal((50, 9)).astype(np.float32))).max() <= 8192


def test_first_draw_frequencies_follow_the_potential():
    """Step 1 with L = 1 draws row i with probability D_i / phi: over 4000 seeds, a chi-square test on the draw counts."""
    from scipy.stats import chisquare
    rng = np.random.default_rng(3)
    x = rng.standard_normal((12, 3)).astype(np.float32)
    P = R.Points(x)
    counts = np.zeros(12)
    for seed in range(4000):
        c0 = R.umulhi(R.u(seed, 0, 0), 12)
        Dm = P.dist([c0])[0]
        phi = int(Dm.sum())
        i = R.draw(Dm, R.umulhi(R.u(seed, 1, 0), phi))
        assert Dm[i] > 0
        counts[i] += 1
        rows, _ = R.seed_rows(x, 2, seed, 1, points=P)
        assert rows == [c0, i]
    # expected frequencies: the average over centre 0 (uniform) of D_i / phi
    want = np.zeros(12)
    for c in range(12):
        Dm = P.dist([c])[0].astype(np.float64)
        want += Dm / Dm.sum() / 12
    assert chisquare(counts, want * 4000).pvalue > 1e-3


def test_ties_between_trials_go_to_the_lowest_trial():
    """Four copies of one point far from a cluster at the origin: once a centre is in the cluster, every trial that draws a copy gives
    the same phi_j, and the centre is the first such trial's row."""
    x = np.zeros((10, 2), np.float32)
    x[6:] = [1.0, 1.0]
    x[:6, 0] = np.arange(6, dtype=np.float32) * 1e-3
    P = R.Points(x)
    seen = 0
    for seed in range(200):
        rows, _ = R.seed_rows(x, 2, seed, 8, points=P)
        if rows[0] >= 6:
            continue
        Dm = P.dist([rows[0]])[0]
        cand = [R.draw(Dm, R.umulhi(R.u(seed, 1, j), int(Dm.sum()))) for j in range(8)]
        far = [j for j in range(8) if cand[j] >= 6]
        if len({cand[j] for j in far}) > 1:
            seen += 1
            assert rows[1] == cand[far[0]]
    assert seen > 10


def test_zero_potential_falls_back_to_uniform_rows():
    x = np.ones((7, 3), np.float32)
    for seed in (0, 1, 99):
        rows, phi = R.seed_rows(x, 5, seed, 2)
        assert phi == 0
        assert rows == [R.umulhi(R.u(seed, 0, 0), 7)] + [R.umulhi(R.u(seed, t, 0), 7) for t in range(1, 5)]
    assert R.seed_rows(np.zeros((4, 2), np.float32), 4, 3, 1)[1] == 0


def test_prefix_property():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((60, 5)).astype(np.float32)
    P = R.Points(x)
    full, _ = R.seed_rows(x, 30, 11, 3, points=P)
    for t in (1, 2, 17, 29):
        assert R.seed_rows(x, t, 11, 3, points=P)[0] == full[:t]
    # with the default L, the trials depend on k
    assert R.default_trials(30) != R.default_trials(2)


def test_api_refusals_without_a_gpu():
    import torch
    from npairloss_b200.torch_api import clustering_metrics
    with pytest.raises(ValueError):
        clustering_metrics(torch.zeros(8, 4), torch.zeros(8), init="kmeans")
    with pytest.raises(ValueError):
        clustering_metrics(torch.zeros(8, 4), torch.zeros(8), n_init=0)
