"""Host references of the evaluator's outputs (include/npair_b200.h, DESIGN 8), shared by its GPU tests: inputs whose similarities are
exact in every operand format, MAP@R / R-Precision / R / rank by a host loop over given similarities, the k-means fixed-point centroid
update, and bitwise comparisons that treat NaN as equal to NaN."""
import numpy as np


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def planted(n, D, n_cls, rng):
    """Entries k/8 with integer k in [-8, 8] (every similarity exact in every operand format), some rows duplicated under another
    label so that negatives tie positives, and a few singleton labels (no positive)."""
    K = rng.integers(-8, 9, size=(n, D)).astype(np.int64)
    lab = rng.integers(0, n_cls, size=n).astype(np.float32)
    for a, b in rng.integers(0, n, size=(n // 6, 2)):
        if a != b:
            K[b] = K[a]
            lab[b] = lab[a] + 1000.0
    lab[rng.integers(0, n, size=5)] = 5000.0 + np.arange(5)
    return K, lab


def map_ref(S, ql, gl, self_offset):
    """Host loop of the header's definitions: (map_r, r_precision, R, rank) per query.  S is exact (int64) or the library's fp32
    similarities; labels compare as floats (-0.0 == +0.0, NaN equals nothing); MAP@R is summed in fp64 in ascending k and divided by R
    last, as the library does."""
    nq, ng = S.shape
    valid = np.ones((nq, ng), bool)
    if self_offset >= 0:
        valid[np.arange(nq), self_offset + np.arange(nq)] = False
    eq = ql[:, None] == gl[None, :]
    same, neg = eq & valid, ~eq & valid
    map_r, r_prec = np.full(nq, np.nan), np.full(nq, np.nan)
    R, rank = same.sum(1).astype(np.int32), np.zeros(nq, np.int32)
    for i in range(nq):
        if R[i] == 0:
            continue
        p = np.sort(S[i][same[i]])[::-1]
        sn = np.sort(S[i][neg[i]])
        neg_ge = len(sn) - np.searchsorted(sn, p, side="left")       # negatives >= p_k
        total, hits = 0.0, 0
        for k in range(1, R[i] + 1):
            pk = k + int(neg_ge[k - 1])
            if pk > R[i]:
                break
            total += k / pk
            hits += 1
        map_r[i], r_prec[i] = total / int(R[i]), hits / int(R[i])
        rank[i] = int((p == p[0]).sum()) + int(neg_ge[0])
    return map_r, r_prec, R, rank


def bits_equal(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    np.testing.assert_array_equal(got[ok].view(np.uint64), want[ok].view(np.uint64))


def check_map(out, ref):
    """Evaluator.map_at_r's outputs against map_ref, bit for bit."""
    m, rp, R, rank = ref
    bits_equal(out["map_r"].cpu().numpy(), m)
    bits_equal(out["r_precision"].cpu().numpy(), rp)
    np.testing.assert_array_equal(out["R"].cpu().numpy(), R)
    np.testing.assert_array_equal(out["rank"].cpu().numpy(), rank)


def sigma_exp(x):
    """e with pre_scale(max|x|) = 2^-e: max|x| = m 2^e, m in [0.5, 1), clamped to [-126, 127] so that 2^-e and 2^e are finite fp32
    values; 0 for an all-zero x (sigma = 1)"""
    return min(max(int(np.frexp(np.float32(np.abs(x).max()))[1]), -126), 127) if np.any(x) else 0


def update_ref(x, assign, C):
    """The header's fixed-point update: int64 sums of rint(x * sigma * 2^32), then (float)(ldexp(sum / count, -32) * 2^e); an empty
    cluster keeps its centroid."""
    e = sigma_exp(x)
    q = np.rint((x * np.float32(2.0 ** -e)).astype(np.float64) * 2.0 ** 32).astype(np.int64)
    k = C.shape[0]
    S = np.zeros((k, x.shape[1]), np.int64)
    np.add.at(S, assign, q)
    cnt = np.bincount(assign, minlength=k)
    out = C.copy()
    ne = cnt > 0
    out[ne] = (np.ldexp(S[ne].astype(np.float64) / cnt[ne, None], -32) * 2.0 ** e).astype(np.float32)
    return out
