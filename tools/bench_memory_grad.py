"""Time of the memory rows' gradient (npair_backward_memory, DESIGN 4.6) on one GPU.

    python tools/bench_memory_grad.py                     # every case below
    python tools/bench_memory_grad.py --cases 512 --repeats 20

Cases: Q = 512 with m in {100, 11318 (the classes of Stanford Online Products: one proxy per class), 16384, 57344}, and Q = 8192 with
m in {8192, 65536}; D = 512, fp16x2, plus bf16x3 at Q = 512, m = 16384; the reference's usage mining block, random unit rows made on
the device from fixed seeds (labels: classes of two rows in the batch, the memory rows drawn from the same classes).  For every case:
--warmup untimed steps, then --repeats steps timed with CUDA events for each of two steps, forward_memory + npair_backward and
forward_memory + npair_backward_memory (alternating, L2 not flushed), and one profiled step that gives phase 7, the memory-row
gradient's kernels.  Its rate counts the MMA work of the memory rows' product, 2 m Q D flops times the format's MMA passes (3 for
fp16x2, 6 for bf16x3).  When m = (W - 1) Q, the workaround a memory gradient used to need is timed as well -- a world-W
external-collectives context fed [x; y] by npair_forward_gathered, with npair_backward_partial's W d_total_half[Q:] as the memory rows'
gradient -- and the normwise difference of that from d_mem_diff is reported.  Prints one JSON line per case with the card's name,
power limit and median SM clock sampled during the timed steps.  Writes nothing.
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

from bench_retrieval_eval import ClockSampler, card  # noqa: E402

D = 512
CASES = {512: [(100, "fp16x2"), (11318, "fp16x2"), (16384, "fp16x2"), (16384, "bf16x3"), (57344, "fp16x2")],
         8192: [(8192, "fp16x2"), (65536, "fp16x2")]}
PASSES = {"fp16x2": 3, "bf16x3": 6}


def timed(steps, warmup, repeats):
    """Median milliseconds of each step, the steps alternating; and the median SM clock."""
    import torch
    for _ in range(warmup):
        for s in steps:
            s()
    torch.cuda.synchronize()
    ms = [[] for _ in steps]
    with ClockSampler() as clk:
        for _ in range(repeats):
            for i, s in enumerate(steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                s()
                e1.record()
                e1.synchronize()
                ms[i].append(e0.elapsed_time(e1))
    return [round(statistics.median(v), 4) for v in ms], clk.median()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", type=int, default=sorted(CASES), choices=sorted(CASES))
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=10)
    args = ap.parse_args()

    import torch
    from npairloss_b200 import capi, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_memory_grad.py needs a CUDA device (the layer has no CPU path)")
    name = card()
    mining = dict(synth.USAGE_MINING)
    prec_of = {"fp16x2": capi.PREC_FP32_FP16X2, "bf16x3": capi.PREC_FP32_BF16X3}
    for Q in args.cases:
        for m, prec in CASES[Q]:
            gen = torch.Generator(device="cuda").manual_seed(20171225 + Q + m)
            xall = torch.randn(Q + m, D, device="cuda", generator=gen)
            xall /= xall.norm(dim=1, keepdim=True)
            lall = torch.cat([torch.arange(Q, device="cuda") // 2, torch.randint(0, Q // 2, (m,), device="cuda", generator=gen)]).float()
            x, lab, y, ly = xall[:Q], lall[:Q], xall[Q:], lall[Q:]
            ctx = capi.Context(capi.make_config(Q, D, sim_precision=prec_of[prec], **mining), memory_rows=m)
            dx, dm = torch.empty_like(x), torch.empty_like(y)

            def plain():
                ctx.forward_memory(x, lab, y, ly, m)
                ctx.backward(1.0, dx)

            def with_mem():
                ctx.forward_memory(x, lab, y, ly, m)
                ctx.backward_memory(1.0, dx, dm)
            (ms_plain, ms_mem), clock = timed([plain, with_mem], args.warmup, args.repeats)
            ctx.profile_enable(True)
            with_mem()
            ph = ctx.profile_read()
            ctx.profile_enable(False)
            flops = 2.0 * m * Q * D * PASSES[prec]
            out = {"Q": Q, "m": m, "D": D, "precision": prec, "ms_step_backward": ms_plain, "ms_step_backward_memory": ms_mem,
                   "ms_phase7_memory_grad": round(ph[7], 4), "ms_phase6_anchor_grad": round(ph[6], 4),
                   "memory_grad_mma_tflops": round(flops / (ph[7] * 1e-3) / 1e12, 1) if ph[7] > 0 else None,
                   "card": name, "sm_clock_mhz_median": clock}
            if m % Q == 0:
                W = 1 + m // Q
                ext = capi.Context(capi.make_config(Q, D, world=W, rank=0, bwd_exchange=1, sim_precision=prec_of[prec], **mining))
                xt, lt = xall.contiguous(), lall.contiguous()
                lh, th = torch.empty(Q, D, device="cuda"), torch.empty(Q + m, D, device="cuda")

                def workaround():
                    ext.forward_gathered(xt, lt)
                    ext.backward_partial(1.0, lh, th)
                (wms,), wclock = timed([workaround], args.warmup, args.repeats)
                workaround()
                with_mem()
                ref = W * th[Q:]
                torch.cuda.synchronize()
                out["workaround"] = {"world": W, "ms_step": wms, "sm_clock_mhz_median": wclock,
                                     "mem_grad_rel_diff": float((dm - ref).norm() / ref.norm())}
                ext.close()
            print(json.dumps(out), flush=True)
            ctx.close()
            del xall, lall, x, lab, y, ly, dx, dm
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
