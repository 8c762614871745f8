"""Exact relative-mining thresholds of a given similarity matrix, and the predicates that say which path each select kernel takes on it.

The thresholds restate DESIGN §4.1 independently of the C++ oracle: the same-label list (AP side) and the diff-label list (AN side) of a
row (LOCAL) or of the whole Q x N block (GLOBAL), the self pair excluded; the order statistic at the reference's fp32 `pos()`; negative
picks clamped to -FLT_MAX.  The unclamped pick is returned too, so a test can assert that its pick is visible through the clamp.

The path predicates restate the size rules of `plan_of` (ctx.cu) and the digit rules of the select kernels (select.cu), so a test can
assert that its data reaches the path it is named after.
"""
import numpy as np

FLT_MAX = np.float32(np.finfo(np.float32).max)
GCAND_ABS_CAP = 32 << 20           # entries per side, whatever Q * N
LSEL_LANE_CAP = 48                 # local_select_kernel: candidates per lane
LSEL_SAME_CAP = 128                # both LOCAL kernels: same-label entries kept per row
GSEL_STAGE = 2048                  # global_select_kernel: staging slots per side and block


def pos(sn, size):
    """0-based rank of the pick in a list of `size` entries (reference .cu:285-287), None when out of range.  SN >= 0 (-0.0 included):
    size - 1 - (int)SN in integer arithmetic; SN < 0: (int)((float)(size - 1) + SN * (float)size), each step rounded to fp32."""
    sn = np.float32(sn)
    if size == 0:
        return None
    if sn >= 0:
        p = size - 1 - int(sn)
    else:
        c = np.float32(size - 1) + sn * np.float32(size)
        if not (-2.0 ** 31 < c < 2.0 ** 31):
            return None
        p = int(c)                                 # truncation toward zero
    return p if 0 <= p < size else None


def clamp(v):
    return np.float32(v) if v >= 0 else -FLT_MAX


def side_masks(lab_rows, lab_cols, self_offset):
    """(same, diff) boolean Q x N masks; the self pair (i, i + self_offset) is in neither."""
    lab_rows, lab_cols = np.asarray(lab_rows, np.float32), np.asarray(lab_cols, np.float32)
    Q = lab_rows.shape[0]
    same = lab_rows[:, None] == lab_cols[None, :]
    diff = ~same
    same[np.arange(Q), np.arange(Q) + self_offset] = False
    diff[np.arange(Q), np.arange(Q) + self_offset] = False
    return same, diff


def _pick(vals, sn):
    p = pos(sn, vals.size)
    if p is None:
        return None, np.float32(np.nan)
    return p, np.partition(vals, p)[p]


def relative_thresholds(S, lab_rows, lab_cols, self_offset, region, identsn, diffsn):
    """Thresholds of both sides for the Q rows of S.  region 0 = GLOBAL (one list per side over the block), 1 = LOCAL (one per row).
    Returns dict(posi, nega: clamped float32[Q]; posi_raw, nega_raw: unclamped; pos_ap, pos_an: the ranks, per row for LOCAL)."""
    S = np.asarray(S, np.float32)
    Q = S.shape[0]
    same, diff = side_masks(lab_rows, lab_cols, self_offset)
    out = {}
    for name, mask, sn in (("posi", same, identsn), ("nega", diff, diffsn)):
        if region == 0:
            p, v = _pick(S[mask], sn)
            raw = np.full(Q, v, np.float32)
            ranks = p
        else:
            raw = np.empty(Q, np.float32)
            ranks = []
            for i in range(Q):
                p, raw[i] = _pick(S[i, mask[i]], sn)
                ranks.append(p)
        out[name + "_raw"] = raw
        out[name] = np.array([clamp(v) for v in raw], np.float32)
        out["pos_ap" if name == "posi" else "pos_an"] = ranks
    return out


# ---- path predicates ----

def gcand_cap(Q, N):
    """Entries per side of the GLOBAL select's candidate lists (plan_of): a chosen first-digit bucket with more entries than this takes
    the three-sweep path, which does not compact."""
    return min(Q * N // 8 + 4096, GCAND_ABS_CAP)


def _digit(vals, bits):
    return np.asarray(vals, np.float32).view(np.uint32) >> np.uint32(32 - bits)


def _order_of_digit(d, bits):
    half = 1 << (bits - 1)                        # digits >= half are the negative floats: descending raw digit in value order
    return np.where(d >= half, 2 * half - 1 - d.astype(np.int64), d.astype(np.int64) + half)


def bucket_of_rank(vals, p, bits):
    """The raw `bits`-bit leading digit (sign, exponent, top mantissa bits) of the bucket that holds 0-based rank p of `vals`, found by
    walking the bucket counts in value order (the rule of raw_digit_of_order), and that bucket's population."""
    half = 1 << (bits - 1)
    hist = np.bincount(_order_of_digit(_digit(vals, bits), bits), minlength=2 * half)
    o = int(np.searchsorted(np.cumsum(hist), p, side="right"))
    raw = 2 * half - 1 - o if o < half else o - half
    return raw, int(hist[o])


def global_bucket(S, lab_rows, lab_cols, self_offset, side, sn):
    """GLOBAL select of one side (0 AP, 1 AN): dict(raw digit, pop = entries of the list in the chosen 11-bit bucket, cap, row_max =
    the most entries of that bucket in one row, row = that row)."""
    S = np.asarray(S, np.float32)
    mask = side_masks(lab_rows, lab_cols, self_offset)[side]
    vals = S[mask]
    raw, pop = bucket_of_rank(vals, pos(sn, vals.size), 11)
    per_row = ((_digit(S, 11) == raw) & mask).sum(axis=1)
    r = int(per_row.argmax())
    return dict(raw=raw, pop=pop, cap=gcand_cap(S.shape[0], S.shape[1]), row_max=int(per_row[r]), row=r)


def local_warp_bins(S, lab_rows, lab_cols, self_offset, sn):
    """local_select_kernel's AN side, per row: the 10-bit bin that holds the wanted rank of the diff-label list, the number of the row's
    entries with that leading digit (all columns: sweep 2 keeps every one of them), and the most of them that one lane sees.  A lane
    with more than LSEL_LANE_CAP takes the slow fallback.  Lanes own 4-column groups (j % 128) // 4 of the 16-byte-load part of the row
    (N rounded down to 128) and single columns of the rest."""
    S = np.asarray(S, np.float32)
    Q, N = S.shape
    diff = side_masks(lab_rows, lab_cols, self_offset)[1]
    n_vec = N & ~127
    j = np.arange(N)
    lane = np.where(j < n_vec, (j % 128) // 4, (j - n_vec) % 32)
    raw = np.empty(Q, np.int64)
    pop = np.empty(Q, np.int64)
    lane_max = np.empty(Q, np.int64)
    for i in range(Q):
        vals = S[i, diff[i]]
        raw[i], _ = bucket_of_rank(vals, pos(sn, vals.size), 10)
        hit = _digit(S[i], 10) == raw[i]
        pop[i] = int(hit.sum())
        lane_max[i] = int(np.bincount(lane[hit], minlength=32).max()) if pop[i] else 0
    return dict(raw=raw, pop=pop, lane_max=lane_max)
