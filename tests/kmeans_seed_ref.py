"""Host reference of the k-means++ seeding rule (npair_eval_kmeans_seed, include/npair_b200.h, DESIGN 8.2): SplitMix64 in Python ints,
the int16 fixed-point rows, exact distances and potentials, and the draws by searchsorted (right) on the int64 cumulative sums."""
import math

import numpy as np

M64 = (1 << 64) - 1
GAMMA = 0x9E3779B97F4A7C15


def splitmix_mix(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def u(seed, t, j):
    """Output number t * 256 + j + 1 of SplitMix64 seeded with seed"""
    return splitmix_mix((seed + (t * 256 + j + 1) * GAMMA) & M64)


def umulhi(a, b):
    return (a * b) >> 64


def default_trials(k):
    return 2 + int(math.floor(math.log(k)))


def quantise(x):
    """q = rint((x * sigma) * 2^13) in fp32 arithmetic, sigma = 2^-max(e, -126) with max|x| = m 2^e, m in [0.5, 1) (pre_scale(max|x|),
    halved where its exponent clamp at 127 would leave |x * sigma| >= 1); 1 for 0"""
    x = np.asarray(x, np.float32)
    amax = np.float32(np.abs(x).max()) if x.size else np.float32(0)
    sigma = np.float32(2.0 ** -max(int(np.frexp(amax)[1]), -126)) if amax > 0 else np.float32(1)
    return np.rint((x * sigma) * np.float32(8192)).astype(np.int64)


class Points:
    """The fixed-point rows with d(., c) for a set of centres: exact, by fp64 products of integers while D * 2^26 < 2^53"""

    def __init__(self, x):
        self.q = quantise(x)
        n, D = self.q.shape
        assert D < 2 ** 27, "the fp64 dot products would not be exact"
        self.qf = self.q.astype(np.float64)
        self.norm = (self.q * self.q).sum(1)
        self.full = self._dist(np.arange(n)) if n <= 5000 else None     # every pair at once for small sets

    def _dist(self, rows):
        dot = (self.qf[rows] @ self.qf.T).astype(np.int64)
        return self.norm[None, :] + self.norm[rows][:, None] - 2 * dot

    def dist(self, rows):
        """[len(rows), n] int64: d(i, c) = ||q_i||^2 + ||q_c||^2 - 2 q_i . q_c"""
        rows = np.asarray(rows, np.int64)
        return self.full[rows] if self.full is not None else self._dist(rows)


def draw(Dmin, target):
    """The smallest i with Dmin[0] + ... + Dmin[i] > target"""
    return int(np.searchsorted(np.cumsum(Dmin.astype(np.uint64)), np.uint64(target), side="right"))


def seed_rows(x, k, seed, local_trials=0, points=None):
    """(rows [k], final phi) of the rule"""
    P = points if points is not None else Points(x)
    n = P.q.shape[0]
    L = local_trials or default_trials(k)
    seed &= M64
    rows = [umulhi(u(seed, 0, 0), n)]
    Dmin = P.dist(rows)[0]
    for t in range(1, k):
        phi = int(Dmin.astype(np.uint64).sum(dtype=np.uint64))
        cand = []
        for j in range(L):
            uj = u(seed, t, j)
            cand.append(umulhi(uj, n) if phi == 0 else draw(Dmin, umulhi(uj, phi)))
        d = np.minimum(P.dist(cand), Dmin[None, :])
        phis = [int(r.astype(np.uint64).sum(dtype=np.uint64)) for r in d]
        jb = min(range(L), key=lambda j: (phis[j], j))
        rows.append(cand[jb])
        Dmin = d[jb]
    return rows, int(Dmin.astype(np.uint64).sum(dtype=np.uint64))


def seed_rows_brute(x, k, seed, local_trials=0):
    """The rule by per-element Python loops over Python ints (tiny sets only)"""
    q = quantise(x).tolist()
    n = len(q)
    L = local_trials or default_trials(k)

    def d(i, j):
        return sum((a - b) ** 2 for a, b in zip(q[i], q[j]))

    rows = [umulhi(u(seed, 0, 0), n)]
    Dm = [d(i, rows[0]) for i in range(n)]
    for t in range(1, k):
        phi = sum(Dm)
        best = None
        for j in range(L):
            uj = u(seed, t, j)
            if phi == 0:
                c = umulhi(uj, n)
            else:
                target, acc, c = umulhi(uj, phi), 0, None
                for i in range(n):
                    acc += Dm[i]
                    if acc > target:
                        c = i
                        break
            pj = sum(min(Dm[i], d(i, c)) for i in range(n))
            if best is None or pj < best[0]:
                best = (pj, c)
        rows.append(best[1])
        Dm = [min(Dm[i], d(i, best[1])) for i in range(n)]
    return rows, sum(Dm)
