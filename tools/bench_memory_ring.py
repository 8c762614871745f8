"""What keeping the cross-batch memory ring in the context saves (npair_forward_ring, DESIGN 4.3.1), on one GPU.

    python tools/bench_memory_ring.py                    # every case
    python tools/bench_memory_ring.py --cases 512:57344 --steps 50 --rounds 3 --torch-q

Library cases: D = 512, fp16x2, the reference's usage mining block, (Q, M) in {(512, 4096), (512, 16384), (512, 57344), (8192, 8192),
(8192, 65536)}.  Batches are random unit rows with classes of two, made on the device from fixed seeds; a pool of eight batches is
cycled.  Two contexts of capacity M step side by side over the same batches:
  ring    npair_forward_ring + npair_backward: the ring in the context, only the stale ring tiles re-split
  memory  npair_forward_memory + npair_backward over a torch ring laid out as NPairLoss's own, then the batch copied into it
Both are first filled to m = M.  Then --check steps compare them bit for bit (tops, gradient) and count the steps whose ring forward
re-split every ring tile (npair_debug_read 13) and those whose fp16x2 pre-scale changed (npair_debug_read 10); then the operand-
preparation phase of one profiled step each (npair_profile phase 1); then --rounds rounds of --steps back-to-back steps, the two
alternating within each round (CUDA events around each run of steps; the memory variant's time includes its ring copy).  Medians per
step are reported.
Torch loop (BASELINE 5.8's): a two-layer MLP (256 -> 1024 -> 512) -> NPairLoss(memory_rows=M, normalize_input=1) -> SGD at Q = 512,
M = 16384: the default module eager with blocking=True and blocking=False, and library_memory=True with the whole step captured with
torch.cuda.graph once the ring is full, replayed.
Prints one JSON line per case with the card's name and power limit and the median SM clock sampled during the timed steps.  Writes
nothing.
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

from bench_async import compare  # noqa: E402
from bench_retrieval_eval import ClockSampler, card  # noqa: E402

D = 512
CASES = [(512, 4096), (512, 16384), (512, 57344), (8192, 8192), (8192, 65536)]
TILE = 32


class TorchRing:
    """NPairLoss's own ring: head = count mod M (Q <= M here)."""

    def __init__(self, torch, M):
        self.M, self.count = M, 0
        self.x = torch.zeros(M, D, device="cuda")
        self.l = torch.zeros(M, device="cuda")

    def push(self, x, lab):
        q, head = x.shape[0], self.count % self.M
        first = min(q, self.M - head)
        self.x[head:head + first].copy_(x[:first]); self.l[head:head + first].copy_(lab[:first])
        if first < q:
            self.x[:q - first].copy_(x[first:]); self.l[:q - first].copy_(lab[first:])
        self.count += q


def lib_case(torch, capi, synth, Q, M, steps, rounds, check):
    gen = torch.Generator(device="cuda").manual_seed(20171225 + Q + M)
    pool = []
    for _ in range(8):
        x = torch.randn(Q, D, device="cuda", generator=gen)
        pool.append((x / x.norm(dim=1, keepdim=True), (torch.arange(Q, device="cuda") // 2).float()))
    cfg = capi.make_config(Q, D, sim_precision=capi.PREC_FP32_FP16X2, **synth.USAGE_MINING)
    ring, mem = capi.Context(cfg, memory_rows=M, ring=True), capi.Context(cfg, memory_rows=M)
    tr = TorchRing(torch, M)
    dx_r, dx_m = torch.empty(Q, D, device="cuda"), torch.empty(Q, D, device="cuda")
    it = {"r": 0, "m": 0}

    def ring_steps(n):
        for _ in range(n):
            x, lab = pool[it["r"] % len(pool)]; it["r"] += 1
            t = ring.forward_ring(x, lab)
            ring.backward(1.0, dx_r)
        return t

    def mem_steps(n):
        for _ in range(n):
            x, lab = pool[it["m"] % len(pool)]; it["m"] += 1
            t = mem.forward_memory(x, lab, tr.x, tr.l, min(tr.count, M))
            mem.backward(1.0, dx_m)
            tr.push(x, lab)
        return t

    fill = -(-M // Q)
    ring_steps(fill); mem_steps(fill)
    # bit for bit, the steps that re-split every ring tile and the pre-scale changes
    bt, nt = -(-Q // TILE), -(-(Q + M) // TILE)
    same, full, changes, tiles = True, 0, 0, []
    scale = ring.debug_read(10, 1)[0]
    for _ in range(check):
        tr_, tm_ = ring_steps(1), mem_steps(1)
        torch.cuda.synchronize()
        same &= tr_ == tm_ and torch.equal(dx_r.view(torch.int32), dx_m.view(torch.int32))
        k = int(ring.debug_read(13, 1 + nt)[0])
        tiles.append(k)
        full += k == nt - bt
        s = ring.debug_read(10, 1)[0]
        changes += int(s != scale)
        scale = s
    prep = {}
    for name, ctx, run in (("ring", ring, ring_steps), ("memory", mem, mem_steps)):
        ctx.profile_enable(True)
        run(1)
        prep[name] = round(ctx.profile_read()[1], 4)
        ctx.profile_enable(False)
    with ClockSampler() as clk:
        res = compare(torch, {"ring": ring_steps, "memory": mem_steps}, steps, rounds)
    same &= it["r"] == it["m"]
    ring.close(); mem.close()
    return {"kind": "library", "Q": Q, "M": M, "m": M, "D": D, "precision": "fp16x2", "steps": steps, "rounds": rounds,
            "per_step_device_ms": {k: v["device_ms"] for k, v in res.items()}, "prep_ms": prep, "bit_equal": bool(same),
            "check_steps": check, "all_tiles_resplit": full, "prescale_changes": changes, "ring_tiles": nt - bt,
            "tiles_resplit_median": statistics.median(tiles), "sm_clock_mhz_median": clk.median()}


def torch_case(torch, torch_api, synth, Q, M, steps, rounds):
    D_in, H = 256, 1024
    gen = torch.Generator(device="cuda").manual_seed(7 + Q)
    x = torch.randn(Q, D_in, device="cuda", generator=gen)
    lab = (torch.arange(Q, device="cuda") // 2).float()

    def make(**kw):
        torch.manual_seed(99)
        net = torch.nn.Sequential(torch.nn.Linear(D_in, H), torch.nn.ReLU(), torch.nn.Linear(H, D)).cuda()
        loss_fn = torch_api.NPairLoss(memory_rows=M, normalize_input=1, **kw, **synth.USAGE_MINING)
        return net, loss_fn, torch.optim.SGD(net.parameters(), lr=0.01)

    def stepper(net, loss_fn, opt):
        def run(n):
            for _ in range(n):
                opt.zero_grad(set_to_none=True)
                loss, _ = loss_fn(net(x), lab)
                loss.backward()
                opt.step()
        return run

    blocking, nonblocking, graphed = make(), make(blocking=False), make(blocking=False, library_memory=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                  # until the ring is full
        stepper(*graphed)(-(-M // Q))
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

    variants = {"default_blocking": stepper(*blocking), "default_nonblocking": stepper(*nonblocking), "library_graph": replay}
    with ClockSampler() as clk:
        res = compare(torch, variants, steps, rounds)
    loss_fn.async_status()
    return {"kind": "torch", "Q": Q, "M": M, "D_in": D_in, "hidden": H, "D": D, "precision": "fp16x2", "steps": steps, "rounds": rounds,
            "per_step": res, "sm_clock_mhz_median": clk.median()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="*", default=None, help="Q:M pairs (default: all)")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--check", type=int, default=20)
    ap.add_argument("--torch-q", nargs="*", type=int, default=[512])
    ap.add_argument("--torch-m", type=int, default=16384)
    args = ap.parse_args()

    import torch
    from npairloss_b200 import capi, synth, torch_api
    if not torch.cuda.is_available():
        raise SystemExit("bench_memory_ring.py needs a CUDA device (the layer has no CPU path)")
    name = card()
    cases = CASES if args.cases is None else [tuple(int(v) for v in c.split(":")) for c in args.cases]
    for Q, M in cases:
        print(json.dumps(dict(lib_case(torch, capi, synth, Q, M, args.steps, args.rounds, args.check), card=name)), flush=True)
        torch.cuda.empty_cache()
    for Q in args.torch_q:
        print(json.dumps(dict(torch_case(torch, torch_api, synth, Q, args.torch_m, args.steps, args.rounds), card=name)), flush=True)


if __name__ == "__main__":
    main()
