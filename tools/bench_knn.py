"""Time of the exact k nearest neighbours (Evaluator.knn, DESIGN 8.3) on one GPU at retrieval-benchmark sizes.

    python tools/bench_knn.py                                  # SOP-like and In-Shop-like shapes, fp16x2 and bf16x3, k = 10, 100, 1000
    python tools/bench_knn.py --shapes sop --precisions fp16x2 --ks 100 --repeats 3

Shapes as in tools/bench_retrieval_eval.py: "sop" = self-retrieval over 60502 x 512, "inshop" = 14218 queries against a disjoint gallery
of 12612, D = 512; random unit vectors made on the device from a fixed seed.  For every shape, format and k: --warmup untimed calls,
then --repeats calls timed with CUDA events (L2 not flushed), and one separate, untimed torch.profiler run of one call that splits its
device time into the similarity sweeps (the store-only GEMM of each row block), the top-k selects and the rest (operand preparation).
Prints one JSON line per (shape, format, k) with the median call milliseconds, the bytes of S stored and re-read per call, the device
memory the call adds (eval_knn_bytes) beside the workspace, and the card's name, power limit and median SM clock sampled during the
timed calls.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_retrieval_eval import PRECS, SHAPES, ClockSampler, card  # noqa: E402


def device_split(f):
    """Device milliseconds of one call of f: the similarity sweeps, the selects and everything else, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    out = {"sweep": 0.0, "select": 0.0, "other": 0.0}
    for e in prof.key_averages():
        if "split_gemm_kernel" in e.key:
            key = "sweep"
        elif "knn_select_kernel" in e.key:
            key = "select"
        elif "npair::" in e.key or e.key.startswith("Memset"):
            key = "other"
        else:
            continue
        out[key] += e.self_device_time_total / 1e3
    return {k: round(v, 4) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["sop", "inshop"], choices=sorted(SHAPES))
    ap.add_argument("--precisions", nargs="+", default=["fp16x2", "bf16x3"], choices=sorted(PRECS))
    ap.add_argument("--ks", nargs="+", type=int, default=[10, 100, 1000])
    ap.add_argument("--block-rows", type=int, default=0)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()

    import torch
    from npairloss_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_knn.py needs a CUDA device (the evaluator has no CPU path)")
    name = card()
    for shape in args.shapes:
        sh = SHAPES[shape]
        nq, ng, D = sh["nq"], sh["ng"], sh["D"]
        gen = torch.Generator(device="cuda").manual_seed(20171225)
        g = torch.randn(ng, D, device="cuda", generator=gen)
        g /= g.norm(dim=1, keepdim=True)
        if sh["self_retrieval"]:
            q, off = g, 0
        else:
            q = torch.randn(nq, D, device="cuda", generator=gen)
            q /= q.norm(dim=1, keepdim=True)
            off = -1
        for pname in args.precisions:
            ev = capi.Evaluator(nq, ng, D, PRECS[pname])
            for k in args.ks:
                def call():
                    return ev.knn(q, g, k, off, block_rows=args.block_rows)
                for _ in range(args.warmup):
                    call()
                torch.cuda.synchronize()
                ms = []
                with ClockSampler() as clk:
                    for _ in range(args.repeats):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        call()
                        e1.record()
                        e1.synchronize()
                        ms.append(e0.elapsed_time(e1))
                split = device_split(call)
                ldS = (ng + 31) // 32 * 32
                print(json.dumps({"shape": shape, "nq": nq, "ng": ng, "D": D, "precision": pname, "k": k,
                                  "block_rows": args.block_rows or 1024,
                                  "ms_median": round(statistics.median(ms), 4), "ms_all": [round(x, 4) for x in ms],
                                  "device_ms_one_call": split,
                                  "s_bytes_stored": 4 * nq * ldS,
                                  "knn_extra_bytes": capi.eval_knn_bytes(ng, k, args.block_rows),
                                  "workspace_bytes": capi.eval_workspace_bytes(nq, ng, D, PRECS[pname]),
                                  "card": name, "sm_clock_mhz_median": clk.median()}), flush=True)
            ev.close()


if __name__ == "__main__":
    main()
