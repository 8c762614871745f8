"""What the asynchronous training step and CUDA-graph replay save (DESIGN 4.4), on one GPU.

    python tools/bench_async.py                      # every case, 200 steps per timing, 5 rounds
    python tools/bench_async.py --steps 50 --rounds 3 --torch-q 512

Library steps: world 1, D = 512, fp16x2, the reference's usage mining block, Q in {512, 2048, 8192} and Q = 512 with m = 16384 memory
rows (random unit rows and classes of two made on the device from fixed seeds), through four variants:
  a  npair_forward (npair_forward_memory) + npair_backward          two host waits per step: the tops, and the ctypes return
  b  npair_forward_backward                                         one host wait per step (no memory form: not run with m > 0)
  c  npair_forward_async (_memory_async) + npair_backward_device_weight     no host wait
  d  a CUDA graph of one step of c, replayed
Torch loop: a two-layer MLP (256 -> 1024 -> 512) -> NPairLoss -> SGD at Q in {512, 2048}, with blocking=True, blocking=False, and the
whole step captured with torch.cuda.graph and replayed.

Each timing runs --steps back-to-back steps: a CUDA event pair gives the device time, a host clock from before the first step to after
a final synchronise gives the wall time, and the host clock when the last step is enqueued gives the enqueue time.  Variants alternate
within each of --rounds rounds; the medians per step are reported.  Every variant's outputs are first checked bit for bit against a.
Prints one JSON line per case with the card's name and power limit and the median SM clock sampled during the case.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_retrieval_eval import ClockSampler, card  # noqa: E402

D = 512
LIB_CASES = [(512, 0), (2048, 0), (8192, 0), (512, 16384)]


def timing(torch, run_steps, steps):
    """(device ms, wall ms, enqueue ms) per step of `steps` back-to-back steps"""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    run_steps(steps)
    t1 = time.perf_counter()
    e1.record()
    e1.synchronize()
    t2 = time.perf_counter()
    return e0.elapsed_time(e1) / steps, (t2 - t0) * 1e3 / steps, (t1 - t0) * 1e3 / steps


def compare(torch, variants, steps, rounds):
    """{variant: {device_ms, wall_ms, enqueue_ms}}: medians over rounds, the variants alternating within each round"""
    res = {k: [] for k in variants}
    for run in variants.values():              # warm-up
        run(3)
    for _ in range(rounds):
        for k, run in variants.items():
            res[k].append(timing(torch, run, steps))
    return {k: {f: round(statistics.median(r[i] for r in v), 5) for i, f in enumerate(("device_ms", "wall_ms", "enqueue_ms"))}
            for k, v in res.items()}


def lib_case(torch, capi, synth, Q, m, steps, rounds):
    gen = torch.Generator(device="cuda").manual_seed(20171225 + Q + m)
    xall = torch.randn(Q + m, D, device="cuda", generator=gen)
    xall /= xall.norm(dim=1, keepdim=True)
    lall = torch.cat([torch.arange(Q, device="cuda") // 2, torch.randint(0, Q // 2, (m,), device="cuda", generator=gen)]).float()
    x, lab, xm, lm = xall[:Q].contiguous(), lall[:Q].contiguous(), xall[Q:].contiguous(), lall[Q:].contiguous()
    cfg = capi.make_config(Q, D, sim_precision=capi.PREC_FP32_FP16X2, **synth.USAGE_MINING)
    ctx = capi.Context(cfg, memory_rows=m)
    dx, tops, lw = torch.empty_like(x), torch.empty(5, device="cuda"), torch.ones(1, device="cuda")

    def a(n):
        for _ in range(n):
            t = ctx.forward_memory(x, lab, xm, lm, m) if m else ctx.forward(x, lab)
            ctx.backward(1.0, dx)
        return t

    def b(n):
        for _ in range(n):
            t = ctx.forward_backward(x, lab, 1.0, dx)
        return t

    def c(n):
        for _ in range(n):
            if m:
                ctx.forward_memory_async(x, lab, xm, lm, m, tops)
            else:
                ctx.forward_async(x, lab, tops)
            ctx.backward_device_weight(lw, dx)

    c(1)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c(1)

    def d(n):
        for _ in range(n):
            g.replay()

    # the outputs of every variant, bit for bit those of a
    ref_tops = torch.tensor(a(1)); ref_dx = dx.clone()
    same = {}
    for k, run in (("b", b), ("c", c), ("d", d)):
        if k == "b" and m:
            continue
        dx.fill_(float("nan"))
        t = run(1)
        torch.cuda.synchronize()
        t = torch.tensor(t) if t is not None else tops.cpu()
        same[k] = bool(torch.equal(t.view(torch.int32), ref_tops.view(torch.int32)) and torch.equal(dx.view(torch.int32), ref_dx.view(torch.int32)))
    variants = {"a": a, "c": c, "d": d} if m else {"a": a, "b": b, "c": c, "d": d}
    with ClockSampler() as clk:
        res = compare(torch, variants, steps, rounds)
    ctx.async_status()
    ctx.close()
    return {"kind": "library", "Q": Q, "m": m, "D": D, "precision": "fp16x2", "steps": steps, "rounds": rounds, "per_step": res,
            "bit_equal_to_a": same, "sm_clock_mhz_median": clk.median()}


def torch_case(torch, torch_api, synth, Q, steps, rounds):
    D_in, H = 256, 1024
    gen = torch.Generator(device="cuda").manual_seed(7 + Q)
    x = torch.randn(Q, D_in, device="cuda", generator=gen)
    lab = (torch.arange(Q, device="cuda") // 2).float()

    def make(blocking):
        torch.manual_seed(99)
        net = torch.nn.Sequential(torch.nn.Linear(D_in, H), torch.nn.ReLU(), torch.nn.Linear(H, D)).cuda()
        loss_fn = torch_api.NPairLoss(blocking=blocking, normalize_input=1, **synth.USAGE_MINING)
        return net, loss_fn, torch.optim.SGD(net.parameters(), lr=0.01)

    def stepper(net, loss_fn, opt):
        def run(n):
            for _ in range(n):
                opt.zero_grad(set_to_none=True)
                loss, _ = loss_fn(net(x), lab)
                loss.backward()
                opt.step()
        return run

    blocking, nonblocking, graphed = make(True), make(False), make(False)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        stepper(*graphed)(3)
    torch.cuda.current_stream().wait_stream(side)
    net, loss_fn, opt = graphed
    g = torch.cuda.CUDAGraph()
    opt.zero_grad(set_to_none=True)
    with torch.cuda.graph(g):
        sloss, _ = loss_fn(net(x), lab)
        sloss.backward()
        opt.step()

    def replay(n):
        for _ in range(n):
            g.replay()

    variants = {"blocking": stepper(*blocking), "nonblocking": stepper(*nonblocking), "graph": replay}
    with ClockSampler() as clk:
        res = compare(torch, variants, steps, rounds)
    nonblocking[1].async_status()
    return {"kind": "torch", "Q": Q, "D_in": D_in, "hidden": H, "D": D, "precision": "fp16x2", "steps": steps, "rounds": rounds,
            "per_step": res, "sm_clock_mhz_median": clk.median()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--lib-q", nargs="*", type=int, default=None, help="library cases by Q (default: all)")
    ap.add_argument("--torch-q", nargs="*", type=int, default=[512, 2048])
    args = ap.parse_args()

    import torch
    from npairloss_b200 import capi, synth, torch_api
    if not torch.cuda.is_available():
        raise SystemExit("bench_async.py needs a CUDA device (the layer has no CPU path)")
    name = card()
    for Q, m in LIB_CASES:
        if args.lib_q is None or Q in args.lib_q:
            print(json.dumps(dict(lib_case(torch, capi, synth, Q, m, args.steps, args.rounds), card=name)), flush=True)
            torch.cuda.empty_cache()
    for Q in args.torch_q:
        print(json.dumps(dict(torch_case(torch, torch_api, synth, Q, args.steps, args.rounds), card=name)), flush=True)


if __name__ == "__main__":
    main()
