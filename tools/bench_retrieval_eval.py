"""Time of the retrieval evaluator (DESIGN 8) on one GPU at retrieval-benchmark sizes.

    python tools/bench_retrieval_eval.py                       # SOP-like and In-Shop-like shapes, fp16x2 and bf16x3
    python tools/bench_retrieval_eval.py --shapes sop --precisions fp16x2 --repeats 3

Shapes: "sop" = self-retrieval over 60502 x 512 (Stanford Online Products' test set), "inshop" = 14218 queries against a disjoint
gallery of 12612, D = 512 (In-Shop).  Inputs are random unit vectors with about 5 rows per label, made on the device from a fixed seed.
For every shape and format: --warmup untimed calls, then --repeats timed rounds of each of the three calls with CUDA events (L2 not
flushed): phase 1 alone (operand preparation + the best-positive sweep), phase 2 alone (operand preparation + the count sweep) and
the one-call rank, and the one-call MAP@R (`map_at_r`: operand preparation + three sweeps + sort + finish).  A separate, untimed
torch.profiler run of one map_at_r call gives the device time of each of its three sweeps (statistics, gather, bucket) and of its other
kernels, and a fp32 torch matmul over --sample queries gives the fraction of the entries that take the bucket sweep's search path
(p_R <= s < p_1 for a negative s).  Prints one JSON line per (shape, format) with median milliseconds, the algorithmic rate
2 * nq * ng * D per sweep over the phase times, and the card's name, power limit and median SM clock sampled during the timed rounds.
Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SHAPES = {"sop": dict(nq=60502, ng=60502, D=512, self_retrieval=True),
          "inshop": dict(nq=14218, ng=12612, D=512, self_retrieval=False)}
PRECS = {"fp16x2": 2, "bf16x3": 0, "bf16": 1}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


class ClockSampler:
    """SM clock (MHz) of GPU 0 every 0.2 s while active."""

    def __init__(self):
        self.samples, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                                     capture_output=True, text=True, timeout=10).stdout.strip()
                self.samples.append(int(out.split()[0]))
            except (OSError, subprocess.SubprocessError, ValueError, IndexError):
                pass
            self._stop.wait(0.2)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join()

    def median(self):
        return statistics.median(self.samples) if self.samples else None


def sweep_times(f):
    """Device milliseconds of each similarity sweep of one call of f (by epilogue) and of everything else, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    names = {16: "stats", 128: "gather", 256: "bucket", 64: "count"}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"split_gemm_kernel<\d+, \w+, (\d+), \d+>", e.key)
        if m:
            key = names.get(int(m.group(1)) & ~32, "other_gemm")
        elif "npair::" in e.key:
            key = "other_kernels"
        elif e.key.startswith("Memset"):
            key = "memset"
        else:
            continue
        out[key] = out.get(key, 0.0) + e.self_device_time_total / 1e3
    return {k: round(v, 4) for k, v in out.items()}


def search_fraction(q, ql, g, gl, off, sample):
    """Share of the valid (query, gallery) entries of `sample` queries that are negatives with p_R <= s < p_1 (fp32 torch matmul)."""
    import torch
    idx = torch.linspace(0, q.shape[0] - 1, min(sample, q.shape[0]), device=q.device).long()
    S = q[idx] @ g.T
    same = ql[idx, None] == gl[None, :]
    valid = torch.ones_like(same)
    if off >= 0:
        valid[torch.arange(len(idx), device=q.device), off + idx] = False
    p1 = torch.where(same & valid, S, torch.full_like(S, -float("inf"))).max(1).values
    pR = torch.where(same & valid, S, torch.full_like(S, float("inf"))).min(1).values
    neg = ~same & valid
    srch = neg & (S >= pR[:, None]) & (S < p1[:, None])
    return float(srch.sum()) / float(valid.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["sop", "inshop"], choices=sorted(SHAPES))
    ap.add_argument("--precisions", nargs="+", default=["fp16x2", "bf16x3"], choices=sorted(PRECS))
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sample", type=int, default=2048, help="queries sampled for the search-path fraction")
    args = ap.parse_args()

    import torch
    from npairloss_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_retrieval_eval.py needs a CUDA device (the evaluator has no CPU path)")
    name = card()
    for shape in args.shapes:
        sh = SHAPES[shape]
        nq, ng, D = sh["nq"], sh["ng"], sh["D"]
        gen = torch.Generator(device="cuda").manual_seed(20171225)
        g = torch.randn(ng, D, device="cuda", generator=gen)
        g /= g.norm(dim=1, keepdim=True)
        gl = torch.randint(0, max(ng // 5, 1), (ng,), device="cuda", generator=gen).float()
        if sh["self_retrieval"]:
            q, ql, off = g, gl, 0
        else:
            q = torch.randn(nq, D, device="cuda", generator=gen)
            q /= q.norm(dim=1, keepdim=True)
            ql = torch.randint(0, max(ng // 5, 1), (nq,), device="cuda", generator=gen).float()
            off = -1
        absmax = float(torch.maximum(q.abs().max(), g.abs().max()))
        for pname in args.precisions:
            ev = capi.Evaluator(nq, ng, D, PRECS[pname])
            cut = ev.best_positive(q, ql, g, gl, absmax, off, 0)
            calls = {"best_positive": lambda: ev.best_positive(q, ql, g, gl, absmax, off, 0),
                     "count": lambda: ev.count(q, g, cut, absmax, off, 0),
                     "rank": lambda: ev.rank(q, ql, g, gl, off),
                     "map_at_r": lambda: ev.map_at_r(q, ql, g, gl, off)}
            for _ in range(args.warmup):
                for f in calls.values():
                    f()
            torch.cuda.synchronize()
            ms = {k: [] for k in calls}
            with ClockSampler() as clk:
                for _ in range(args.repeats):
                    for k, f in calls.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        f()
                        e1.record()
                        e1.synchronize()
                        ms[k].append(e0.elapsed_time(e1))
            rank = ev.rank(q, ql, g, gl, off)
            r1 = float(((rank >= 1) & (rank <= 1)).float().mean())
            mp = ev.map_at_r(q, ql, g, gl, off)
            has = mp["R"] > 0
            map_r = float(mp["map_r"][has].mean())
            sum_r = int(mp["R"].long().sum())
            sweeps = sweep_times(lambda: ev.map_at_r(q, ql, g, gl, off))
            ev.close()
            frac = search_fraction(q, ql, g, gl, off, args.sample)
            flop = 2.0 * nq * ng * D
            med = {k: statistics.median(v) for k, v in ms.items()}
            print(json.dumps({"shape": shape, "nq": nq, "ng": ng, "D": D, "precision": pname,
                              "symmetric_tiles": bool(sh["self_retrieval"]),
                              "ms_median": {k: round(v, 4) for k, v in med.items()},
                              "ms_all": {k: [round(x, 4) for x in v] for k, v in ms.items()},
                              "algorithmic_tflops_per_sweep": {k: round(flop / (med[k] * 1e-3) / 1e12, 1) for k in ("best_positive", "count")},
                              "recall_at_1": round(r1, 5), "map_at_r": round(map_r, 5),
                              "map_at_r_device_ms_by_kernel": sweeps, "search_path_fraction_sampled": round(frac, 5),
                              "map_at_r_extra_bytes": capi.eval_map_at_r_bytes(nq, sum_r),
                              "workspace_bytes": capi.eval_workspace_bytes(nq, ng, D, PRECS[pname]),
                              "card": name, "sm_clock_mhz_median": clk.median()}), flush=True)


if __name__ == "__main__":
    main()
