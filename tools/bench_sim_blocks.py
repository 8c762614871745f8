"""Step time of the row-block similarity mode (NPAIR_SIM_BLOCK_ROWS, DESIGN 4.2) next to the materialised path, one GPU.

    python tools/bench_sim_blocks.py --batch 8192 --dim 512 --heights 0 1024 4096 --rounds 3
    python tools/bench_sim_blocks.py --batch 196608 --dim 256 --heights 2048 16896 --steps 5 --warmup 2

Inputs are bench.py's synthetic ones (B/2 classes x 2, noise 2.5, seed 20171225 + 5, fp16x2).  For every round, a context of each
height in turn is created, warmed up and timed with CUDA events around --steps npair_forward_backward calls (L2 not flushed), so
the heights alternate.  A height of 0 is the materialised path; it needs 4*B*B bytes for S.  Prints one JSON line per height:
ms per step of each round, workspace bytes, per-phase times of one profiled step, and whether tops and gradient are bitwise
those of the first height.  Writes nothing.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PHASES = ["fwd_allgather", "operand_prep", "sim_gemm", "thresholds_select", "row_pass_finalize", "weight_build", "grad_gemm",
          "grad_gemm_T", "bwd_exchange"]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--heights", type=int, nargs="+", default=[0, 1024])
    ap.add_argument("--mining", default="usage", choices=["usage", "rand"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=1)
    args = ap.parse_args()

    import numpy as np
    import torch
    from npairloss_b200 import capi, synth

    assert torch.cuda.is_available(), "needs an H100 (the library has no CPU fallback)"
    B, D = args.batch, args.dim
    mining = dict(synth.USAGE_MINING if args.mining == "usage" else synth.DEFAULT_MINING)
    x, lab = synth.make_inputs(B, D, 20171225 + 5, noise=2.5)
    d_x, d_l = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    del x
    d_g = torch.empty_like(d_x)
    res = {h: dict(ms=[], same_as_first=None) for h in args.heights}
    ref = None
    for _ in range(args.rounds):
        for h in args.heights:
            cfg = capi.make_config(B, D, sim_block_rows=h, **mining)
            res[h]["workspace_bytes"] = int(capi.lib().npair_workspace_bytes(C.byref(cfg)))
            ctx = capi.Context(cfg)
            for _ in range(args.warmup):
                tops = ctx.forward_backward(d_x, d_l, 1.0, d_g)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                tops = ctx.forward_backward(d_x, d_l, 1.0, d_g)
            e1.record()
            torch.cuda.synchronize()
            res[h]["ms"].append(e0.elapsed_time(e1) / args.steps)
            if "phase_ms" not in res[h]:
                ctx.profile_enable(True)
                ctx.forward_backward(d_x, d_l, 1.0, d_g)
                res[h]["phase_ms"] = dict(zip(PHASES, ctx.profile_read()))
                ctx.profile_enable(False)
            ctx.close()
            torch.cuda.synchronize()
            if ref is None:
                ref = (np.asarray(tops, np.float32), d_g.clone())
            same = bool(np.array_equal(np.asarray(tops, np.float32).view(np.uint32), ref[0].view(np.uint32))
                        and torch.equal(d_g.view(torch.int32), ref[1].view(torch.int32)))
            res[h]["same_as_first"] = same if res[h]["same_as_first"] is None else (res[h]["same_as_first"] and same)
            res[h]["tops"] = [float(t) for t in tops]
    gpu = card()
    for h in args.heights:
        r = res[h]
        print(json.dumps({"batch": B, "dim": D, "mining": args.mining, "sim_block_rows": h, "workspace_bytes": r["workspace_bytes"],
                          "ms_per_step": r["ms"], "samples_per_s": B / (min(r["ms"]) * 1e-3), "phase_ms": r["phase_ms"],
                          "tops": r["tops"], "bitwise_equal_to_first_height": r["same_as_first"], "steps": args.steps,
                          "warmup": args.warmup, "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
