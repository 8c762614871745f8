"""Time of the evaluator's k-means (npair_eval_kmeans, DESIGN 8.2) on one GPU at the clustering protocol's sizes.

    python tools/bench_clustering.py                               # CUB-, Cars- and SOP-like shapes, fp16x2 and bf16x3
    python tools/bench_clustering.py --shapes sop --precisions fp16x2 --repeats 3
    python tools/bench_clustering.py --init kmeans++ --n-init 2      # k-means++ seeding (npair_eval_kmeans_seed) before each run

Shapes (k = the number of test classes): "cub" = 5924 x 512, k = 100; "cars" = 8131 x 512, k = 98; "sop" = 60502 x 512, k = 11316.
Inputs are random unit vectors with about 5 rows per label (a label's rows scattered around a random unit centre), made on the device
from a fixed seed.  For every shape and format: --warmup untimed calls, then --repeats timed calls of --iters assignment sweeps each
with CUDA events, reported per iteration (the call's one host synchronisation per iteration included); a separate torch.profiler run
of one call gives the device time per iteration of the EPI_ARGMAX sweep, of the assignment decode with its int64 atomics
(km_assign_kernel) and of the centroid update, and the other kernels and memsets.  Prints one JSON line per (shape, format) with the
card's name, power limit and median SM clock sampled during the timed calls.  --init kmeans++ seeds every run with
Evaluator.kmeans_seed (default trials, seed = the run's index) instead of a random permutation, and --n-init runs that many seedings and
Lloyd calls per repeat; the seeding time (host clock around the call, which ends in its one synchronisation) is reported apart from the
Lloyd time, as seed_ms (median over every seeding) and lloyd_ms (median per call), with the device time per seeding step of its two kernels from a
separate torch.profiler run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_retrieval_eval import ClockSampler, card  # noqa: E402

SHAPES = {"cub": dict(n=5924, k=100, D=512), "cars": dict(n=8131, k=98, D=512), "sop": dict(n=60502, k=11316, D=512)}
PRECS = {"fp16x2": 2, "bf16x3": 0, "bf16": 1}


def make_set(n, D, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    labels = (torch.arange(n, device="cuda") // 5)[torch.randperm(n, device="cuda", generator=g)]
    centres = torch.randn(n // 5 + 1, D, device="cuda", generator=g)
    centres /= centres.norm(dim=1, keepdim=True)
    x = centres[labels] + 0.05 * torch.randn(n, D, device="cuda", generator=g)
    return (x / x.norm(dim=1, keepdim=True)).contiguous(), labels


def phase_times(f, iters):
    """Device milliseconds per iteration of the sweep, the decode, the update and the rest of one call of f, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if re.search(r"split_gemm_kernel<\d+, \w+, 512, \d+>", e.key):
            key = "sweep"
        elif "km_assign_kernel" in e.key:
            key = "assign"
        elif "km_update_kernel" in e.key:
            key = "update"
        elif "npair::" in e.key:
            key = "other_kernels"
        elif e.key.startswith("Memset") or e.key.startswith("Memcpy"):
            key = "memset_memcpy"
        else:
            continue
        out[key] = out.get(key, 0.0) + e.self_device_time_total / 1e3
    return {k: round(v / iters, 4) for k, v in out.items()}


def seed_phase_times(f, steps):
    """Device microseconds per step of the k-means++ distance and update kernels, and the rest, in one call of f (torch.profiler)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        key = "distance" if "kms_distance_kernel" in e.key else "update" if "kms_update_kernel" in e.key else "other"
        out[key] = out.get(key, 0.0) + e.self_device_time_total
    return {k: round(v / steps, 2) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["cub", "cars", "sop"], choices=sorted(SHAPES))
    ap.add_argument("--precisions", nargs="+", default=["fp16x2", "bf16x3"], choices=sorted(PRECS))
    ap.add_argument("--iters", type=int, default=10, help="assignment sweeps per call (max_iter; a call may converge earlier)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--init", choices=["random", "kmeans++"], default="random")
    ap.add_argument("--n-init", type=int, default=1, help="seedings and Lloyd calls per repeat")
    args = ap.parse_args()
    import torch
    from npairloss_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_clustering needs a GPU")
    name = card()
    for sname in args.shapes:
        s = SHAPES[sname]
        n, k, D = s["n"], s["k"], s["D"]
        x, _ = make_set(n, D, 20261016)
        for pname in args.precisions:
            ev = capi.Evaluator(n, k, D, PRECS[pname])
            try:
                def init_rows(r):
                    if args.init == "random":
                        return torch.randperm(n, generator=torch.Generator().manual_seed(r))[:k].tolist()
                    return ev.kmeans_seed(x, k, r)[0]
                rows0 = init_rows(0)
                call = lambda: ev.kmeans(x, k, rows0, args.iters)  # noqa: E731
                for _ in range(args.warmup):
                    call()
                torch.cuda.synchronize()
                per_iter, lloyd, seeding, its = [], [], [], None
                with ClockSampler() as clk:
                    for _ in range(args.repeats):
                        for r in range(args.n_init):
                            t0 = time.perf_counter()
                            rows = init_rows(r)
                            seeding.append((time.perf_counter() - t0) * 1e3)
                            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            a.record()
                            res = ev.kmeans(x, k, rows, args.iters)
                            b.record()
                            torch.cuda.synchronize()
                            its = res["iterations"]
                            lloyd.append(a.elapsed_time(b))
                            per_iter.append(lloyd[-1] / its)
                phases = phase_times(call, call()["iterations"])
                seed_phases = seed_phase_times(lambda: init_rows(0), k) if args.init == "kmeans++" else None
            finally:
                ev.close()
            pairs = n * k
            res = {"shape": sname, "precision": pname, "n": n, "k": k, "D": D, "init": args.init, "n_init": args.n_init,
                   "seed_ms": round(statistics.median(seeding), 3), "seed_ms_all": [round(t, 3) for t in seeding],
                   "seed_device_us_per_step": seed_phases, "lloyd_ms": round(statistics.median(lloyd), 3), "iterations": its,
                   "ms_per_iteration": round(statistics.median(per_iter), 4), "ms_per_iteration_all": [round(t, 4) for t in per_iter],
                   "device_ms_per_iteration": phases, "point_centroid_pairs": pairs,
                   "sweep_pairs_per_s": round(pairs / (phases.get("sweep", 0.0) / 1e3), 1) if phases.get("sweep") else None,
                   "tiles": -(-n // 128) * -(-k // 256), "card": name, "sm_clock_mhz_median": clk.median()}
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
