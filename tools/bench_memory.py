"""Time of a training step with a cross-batch memory (npair_forward_memory + npair_backward, DESIGN 4.3) on one GPU.

    python tools/bench_memory.py                         # Q = 8192 and the XBM-like Q = 512, D = 512, fp16x2
    python tools/bench_memory.py --cases 512 --repeats 20

Cases: Q = 8192 with m in {0, 8192, 32768, 65536} memory rows, and Q = 512 with m in {0, 4096, 16384, 57344}; D = 512, fp16x2, the
reference's usage mining block, random unit rows made on the device from fixed seeds (labels: classes of two rows in the batch, the
memory drawn from the same classes).  One memory context per Q, created with the largest m as its capacity.  For every m: --warmup
untimed steps, then --repeats steps timed with CUDA events (forward with its host wait for the tops, then the backward; L2 not flushed),
and one more step with npair_profile that splits its device time into the layer's phases.  When m = (W - 1) Q, the same step is also
timed through the workaround a memory used to need -- a world-W external-collectives context fed [x; x_mem] by npair_forward_gathered,
with npair_backward_partial's d_local_half + W d_total_half[:Q] as the gradient -- and its outputs are compared with the memory step's
(tops bit for bit, gradient normwise).  Prints one JSON line per (Q, m) with the median step milliseconds, the phases, the context's
device memory, and the card's name, power limit and median SM clock sampled during the timed steps.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_retrieval_eval import ClockSampler, card  # noqa: E402

CASES = {8192: (0, 8192, 32768, 65536), 512: (0, 4096, 16384, 57344)}
D = 512
PHASES = ["allgather", "prep", "sim_gemm", "thresholds", "row_pass", "weights", "grad_gemm", "grad_gemm_T", "bwd_exchange"]


def timed(step, warmup, repeats):
    import torch
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ms = []
    with ClockSampler() as clk:
        for _ in range(repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
    return ms, clk.median()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", type=int, default=sorted(CASES, reverse=True), choices=sorted(CASES))
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--no-workaround", action="store_true")
    args = ap.parse_args()

    import torch
    from npairloss_b200 import capi, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_memory.py needs a CUDA device (the layer has no CPU path)")
    name = card()
    mining = dict(synth.USAGE_MINING)
    for Q in args.cases:
        M = max(CASES[Q])
        gen = torch.Generator(device="cuda").manual_seed(20171225 + Q)
        xall = torch.randn(Q + M, D, device="cuda", generator=gen)
        xall /= xall.norm(dim=1, keepdim=True)
        lall = torch.cat([torch.arange(Q, device="cuda") // 2,
                          torch.randint(0, Q // 2, (M,), device="cuda", generator=gen)]).float()
        x, lab, xm, lm = xall[:Q], lall[:Q], xall[Q:], lall[Q:]
        cfg = capi.make_config(Q, D, sim_precision=capi.PREC_FP32_FP16X2, **mining)
        ctx = capi.Context(cfg, memory_rows=M)
        dx = torch.empty_like(x)
        for m in CASES[Q]:
            def step():
                ctx.forward_memory(x, lab, xm, lm, m)
                ctx.backward(1.0, dx)
            ms, clock = timed(step, args.warmup, args.repeats)
            ctx.profile_enable(True)
            tops = ctx.forward_memory(x, lab, xm, lm, m)
            ctx.backward(1.0, dx)
            phases = dict(zip(PHASES, (round(v, 4) for v in ctx.profile_read())))
            ctx.profile_enable(False)
            torch.cuda.synchronize()
            out = {"Q": Q, "m": m, "D": D, "precision": "fp16x2", "ms_median": round(statistics.median(ms), 4),
                   "ms_all": [round(v, 4) for v in ms], "phases_ms": phases,
                   "workspace_bytes": capi.memory_workspace_bytes(cfg, M), "card": name, "sm_clock_mhz_median": clock}
            W = 1 + m // Q
            if not args.no_workaround and m and m % Q == 0:
                ext = capi.Context(capi.make_config(Q, D, world=W, rank=0, bwd_exchange=1, sim_precision=capi.PREC_FP32_FP16X2, **mining))
                xt, lt = xall[:Q + m].contiguous(), lall[:Q + m].contiguous()
                lh = torch.empty(Q, D, device="cuda")
                th = torch.empty(Q + m, D, device="cuda")

                def wstep():
                    ext.forward_gathered(xt, lt)
                    ext.backward_partial(1.0, lh, th)
                wms, wclock = timed(wstep, args.warmup, args.repeats)
                wtops = ext.forward_gathered(xt, lt)
                ext.backward_partial(1.0, lh, th)
                g = lh + W * th[:Q]
                torch.cuda.synchronize()
                rel = float((dx - g).norm() / g.norm())
                ext.close()
                out["workaround"] = {"world": W, "ms_median": round(statistics.median(wms), 4), "sm_clock_mhz_median": wclock,
                                     "tops_bit_equal": struct.pack("5f", *tops) == struct.pack("5f", *wtops),
                                     "grad_rel_diff": rel}
            print(json.dumps(out), flush=True)
        ctx.close()
        del xall, lall, x, lab, xm, lm, dx
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
