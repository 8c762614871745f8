"""What per-anchor loss weights (npair_set_anchor_io, DESIGN 4.5) cost the training step, on one GPU.

    python tools/bench_anchor_weights.py                    # Q = 8192 (HL) and Q = 512, D = 512, fp16x2 and bf16x3
    python tools/bench_anchor_weights.py --steps 50 --rounds 3

Library step npair_forward_async + npair_backward_device_weight (no host wait), world 1, the reference's usage mining block, random
unit rows in classes of two made on the device from a fixed seed, three variants:
  none      no anchor IO (the unweighted step)
  weights   Q anchor weights in [0, 1], uniform with exact zeros and ones
  weights+  the weights and the per-anchor loss output
Each timing runs --steps back-to-back steps between a CUDA event pair; variants alternate within each of --rounds rounds and the
median per step is reported with the min and max of the rounds.  The weighted step's outputs are first checked against the unweighted
step: w = 1 must give the same bits.  Prints one JSON line per case with the card's name and power limit and the median SM clock
sampled during the case.  Writes nothing.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--q", type=int, nargs="*", default=[8192, 512])
    ap.add_argument("--precision", nargs="*", default=["fp16x2", "bf16x3"])
    a = ap.parse_args()
    import torch

    from npairloss_b200 import capi, synth
    assert torch.cuda.is_available(), "bench_anchor_weights times the GPU step: it needs an H100"
    precs = {"fp16x2": capi.PREC_FP32_FP16X2, "bf16x3": capi.PREC_FP32_BF16X3}
    name = card()
    for prec in a.precision:
        for Q in a.q:
            g = torch.Generator(device="cuda").manual_seed(Q)
            x = torch.nn.functional.normalize(torch.randn(Q, D, device="cuda", generator=g), dim=1).contiguous()
            lab = (torch.arange(Q, device="cuda") // 2).float()
            w = torch.rand(Q, device="cuda", generator=g)
            w[::7] = 0.0
            w[1::7] = 1.0
            rl = torch.empty(Q, device="cuda")
            ctx = capi.Context(capi.make_config(Q, D, sim_precision=precs[prec], **synth.USAGE_MINING))
            tops = torch.empty(5, device="cuda")
            dx = torch.empty_like(x)
            lw = torch.ones(1, device="cuda")
            io = {"none": (None, None), "weights": (w, None), "weights+": (w, rl)}

            def step():
                ctx.forward_async(x, lab, tops)
                ctx.backward_device_weight(lw, dx)

            # w = 1 is the unweighted step, bit for bit
            outs = []
            for iw in (None, torch.ones(Q, device="cuda")):
                ctx.set_anchor_io(iw, None)
                step()
                torch.cuda.synchronize()
                outs.append((tops.clone(), dx.clone()))
            assert torch.equal(outs[0][0].view(torch.int32), outs[1][0].view(torch.int32))
            assert torch.equal(outs[0][1].view(torch.int32), outs[1][1].view(torch.int32))
            times = {k: [] for k in io}
            with ClockSampler() as clk:
                for k in io:                         # warm-up
                    ctx.set_anchor_io(*io[k])
                    for _ in range(5):
                        step()
                torch.cuda.synchronize()
                for _ in range(a.rounds):
                    for k in io:
                        ctx.set_anchor_io(*io[k])
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(a.steps):
                            step()
                        e1.record()
                        e1.synchronize()
                        times[k].append(e0.elapsed_time(e1) / a.steps)
            ctx.async_status()
            ctx.close()
            print(json.dumps({"case": f"Q{Q} D{D} {prec}", "card": name, "sm_clock_mhz_median": clk.median(), "steps": a.steps,
                              "rounds": a.rounds,
                              **{f"{k}_ms": {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}
                                 for k, v in times.items()}}), flush=True)


if __name__ == "__main__":
    main()
