"""Time of the L2Normalize producer (npair_l2normalize_forward / _backward) on one GPU, alone and inside a training step, for one or
more builds of the library, alternated in one run.

    python tools/bench_l2normalize.py                                  # the library of this tree
    python tools/bench_l2normalize.py --libs a/libnpair_b200.so b/libnpair_b200.so --rounds 3

Each (library, round) is a subprocess of its own (the library is chosen when capi is imported), and the libraries alternate round by
round, so that a drift of the card's clocks falls on all of them alike.  Every subprocess measures:
  - standalone: the forward and the backward at 8192 x 512 and 60502 x 512 (Gaussian rows made on the device from fixed seeds), on
    ordinary rows and with one row in 64 scaled by 2^100 or 2^-100 (rows the rescued pass redoes).  --launches back-to-back calls of
    the C ABI into preallocated buffers between one pair of CUDA events, --repeats times; the median microseconds per call and the
    HBM bytes per call over it.
  - step_kernels: the HL step (B = 8192, D = 512, usage mining, fp16x2, normalize_input = 1; rows of norm about 7) under
    torch.profiler: the mean device time of the step's own l2norm_fwd_kernel and l2norm_bwd_kernel launches.
  - step_ms: the median time of the same step with normalize_input = 1 and = 0, --launches steps between one pair of events.
Prints one JSON line per subprocess (with the card's name and power limit) and one summary line of medians over the rounds.
Writes nothing."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def worker(a):
    import torch

    from bench_retrieval_eval import card
    from npairloss_b200 import capi, synth

    L, st = capi.lib(), torch.cuda.current_stream().cuda_stream

    def per_call_us(fn):
        for _ in range(a.warmup):
            fn()
        ts = []
        for _ in range(a.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3 / a.launches)
        return statistics.median(ts)

    out = {"lib": capi.LIB_PATH, "card": card(), "standalone": []}
    for R in (8192, 60502):
        D = 512
        g = torch.Generator(device="cuda").manual_seed(R)
        x = torch.randn(R, D, device="cuda", generator=g)
        dy = torch.randn(R, D, device="cuda", generator=g)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        inv = torch.empty(R, device="cuda")
        for rows in ("ordinary", "rescued 1/64"):
            if rows != "ordinary":
                x[0::128] *= 2.0 ** 100
                x[64::128] *= 2.0 ** -100
            fwd = per_call_us(lambda: L.npair_l2normalize_forward(x.data_ptr(), R, D, y.data_ptr(), inv.data_ptr(), st))
            bwd = per_call_us(lambda: L.npair_l2normalize_backward(y.data_ptr(), inv.data_ptr(), dy.data_ptr(), R, D, dx.data_ptr(), st))
            out["standalone"].append({"rows": R, "D": D, "input": rows, "fwd_us": fwd, "bwd_us": bwd,
                                      "fwd_GBps": 2 * R * D * 4 / fwd / 1e3, "bwd_GBps": 3 * R * D * 4 / bwd / 1e3})
    B, D = 8192, 512
    xh, lab = synth.make_inputs(B, D, seed=20171225)
    xt, lt = torch.from_numpy(xh * 7.0).cuda(), torch.from_numpy(lab).cuda()
    gd = torch.empty_like(xt)
    ctxs = {n: capi.Context(capi.make_config(B, D, normalize_input=n, **synth.USAGE_MINING)) for n in (1, 0)}

    def step(n):
        ctxs[n].forward(xt, lt)
        ctxs[n].backward(1.0, gd)

    out["step_ms"] = {f"normalize_input={n}": per_call_us(lambda: step(n)) / 1e3 for n in (1, 0)}
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        step(1)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            step(1)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k in ("l2norm_fwd_kernel", "l2norm_bwd_kernel"):
            if k in ev.name:
                kern.setdefault(k, []).append(ev.time_range.elapsed_us())
    out["step_kernels_us"] = {k: {"calls": len(v), "mean_us": sum(v) / len(v)} for k, v in kern.items()}
    for c in ctxs.values():
        c.close()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="*", default=None, help="libnpair_b200.so builds to compare (default: this tree's)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=15)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)
    libs = [os.path.abspath(p) for p in a.libs] if a.libs else [None]
    runs = {str(p): [] for p in libs}
    for _ in range(a.rounds):
        for p in libs:
            env = dict(os.environ)
            if p:
                env["NPAIR_LIB"] = p
            args = [sys.executable, os.path.abspath(__file__), "--worker", "--warmup", str(a.warmup), "--repeats", str(a.repeats),
                    "--launches", str(a.launches)]
            r = subprocess.run(args, env=env, capture_output=True, text=True, check=True)
            line = r.stdout.strip().splitlines()[-1]
            print(line, flush=True)
            runs[str(p)].append(json.loads(line))
    summary = {}
    for p, rs in runs.items():
        s = {}
        for i, c in enumerate(rs[0]["standalone"]):
            for k in ("fwd_us", "bwd_us"):
                s[f"{c['rows']}x{c['D']} {c['input']} {k}"] = statistics.median(r["standalone"][i][k] for r in rs)
        for k in rs[0]["step_ms"]:
            s[f"HL step ms {k}"] = statistics.median(r["step_ms"][k] for r in rs)
        for k in rs[0]["step_kernels_us"]:
            s[f"HL step {k} us"] = statistics.median(r["step_kernels_us"][k]["mean_us"] for r in rs)
        summary[p] = s
    print(json.dumps({"summary": summary, "card": runs[str(libs[0])][0]["card"]}))


if __name__ == "__main__":
    main()
