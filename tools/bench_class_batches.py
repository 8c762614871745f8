"""Time of hard negative class mining (Evaluator.class_batches, DESIGN 8.4) on one GPU at training-set sizes.

    python tools/bench_class_batches.py                        # SOP-sized and 40 000-class shapes, fp16x2
    python tools/bench_class_batches.py --shapes sop --ns 60 --precisions fp16x2 bf16x3 --repeats 3

Shapes: "sop" = the 11 318 training classes of Stanford Online Products, every class in each pool (P = C), b = 189 = ceil(11 318 / 60)
batches (each class appears once on average at n = 60); "c40k" = 40 000 classes, pools of NPAIR_EVAL_CLASS_POOL_MAX = 16 384, b = 132
(one batch per SM of an H100 SXM).  D = 512, random unit class embeddings made on the
device and random pools on the host, both from fixed seeds.  For every shape, format and n: --warmup untimed calls, then --repeats calls
timed with CUDA events (L2 not flushed; the call's host-side pool checks and upload included), and one separate, untimed torch.profiler
run of one call that splits its device time into the store-only similarity sweep, the greedy kernel and the rest (operand preparation,
the pool upload).  Prints one JSON line per (shape, format, n) with the median call milliseconds, the device memory the call adds
(eval_class_batches_bytes) beside the workspace, and the card's name, power limit and median SM clock sampled during the timed calls.
Writes nothing.
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

from bench_retrieval_eval import PRECS, ClockSampler, card  # noqa: E402

SHAPES = {"sop": {"C": 11318, "P": 11318, "b": 189, "ns": (60, 512)},
          "c40k": {"C": 40000, "P": 16384, "b": 132, "ns": (60, 4096)}}
D = 512


def device_split(f):
    """Device milliseconds of one call of f: the similarity sweep, the greedy kernel and everything else, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    out = {"sweep": 0.0, "greedy": 0.0, "other": 0.0}
    for e in prof.key_averages():
        if "split_gemm_kernel" in e.key:
            key = "sweep"
        elif "class_batch_kernel" in e.key:
            key = "greedy"
        elif "npair::" in e.key or e.key.startswith("Memset") or e.key.startswith("Memcpy"):
            key = "other"
        else:
            continue
        out[key] += e.self_device_time_total / 1e3
    return {k: round(v, 4) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["sop", "c40k"], choices=sorted(SHAPES))
    ap.add_argument("--precisions", nargs="+", default=["fp16x2"], choices=sorted(PRECS))
    ap.add_argument("--ns", nargs="+", type=int, default=None, help="classes per batch (default: the shape's two)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch
    from npairloss_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_class_batches.py needs a CUDA device (the evaluator has no CPU path)")
    name = card()
    for shape in args.shapes:
        sh = SHAPES[shape]
        C, P, b = sh["C"], sh["P"], sh["b"]
        gen = torch.Generator(device="cuda").manual_seed(20171225)
        x = torch.randn(C, D, device="cuda", generator=gen)
        x /= x.norm(dim=1, keepdim=True)
        rng = np.random.default_rng(20171225)
        pools = np.stack([rng.permutation(C)[:P] for _ in range(b)]).astype(np.int32)
        for pname in args.precisions:
            ev = capi.Evaluator(C, C, D, PRECS[pname])
            for n in args.ns or sh["ns"]:
                def call():
                    return ev.class_batches(x, pools, n)
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
                print(json.dumps({"shape": shape, "C": C, "P": P, "b": b, "n": n, "D": D, "precision": pname,
                                  "ms_median": round(statistics.median(ms), 4), "ms_all": [round(v, 4) for v in ms],
                                  "device_ms_one_call": split,
                                  "class_batches_extra_bytes": capi.eval_class_batches_bytes(C, P, b),
                                  "workspace_bytes": capi.eval_workspace_bytes(C, C, D, PRECS[pname]),
                                  "card": name, "sm_clock_mhz_median": clk.median()}), flush=True)
            ev.close()


if __name__ == "__main__":
    main()
