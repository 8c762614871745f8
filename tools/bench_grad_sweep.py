"""Where the fused gradient kernel's time goes: the gradient phase of the headline step (HL: B = 8192, D = 512, one GPU) timed in
builds that each leave one part of the kernel out (NPAIR_GRAD_PROBE, grad_fused.cuh).  The probes compute garbage; only their time
means something.

    python tools/bench_grad_sweep.py --build                 # compile one library per probe into --lib-dir (needs a built tree)
    python tools/bench_grad_sweep.py [--precisions fp16x2 bf16x3] [--steps 20]

Probes: 0 as is; 1 constant weight fragments (no weight build: loads, MMAs and drain kept); 2 no MMAs (loads, weight build and
drain kept).  Each probe runs in a process of its own (NPAIR_LIB) and times the gradient phase of the backward (npair_profile_read
phase 6, CUDA events) over --steps forward + backward steps, the L2 flushed before each.  Prints one JSON line per (format, probe)
with the median gradient-phase milliseconds and the card's name, power limit and median SM clock during the timed steps.  Writes
nothing outside --lib-dir.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

PROBES = {0: "as_is", 1: "no_weight_build", 2: "no_mma"}
CSRC = os.path.join(ROOT, "npairloss_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def build(lib_dir):
    """libnpair_probe<k>.so per probe: gemm.cu recompiled with -DNPAIR_GRAD_PROBE=k, linked with the tree's other objects."""
    os.makedirs(lib_dir, exist_ok=True)
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    flags = arch + ["-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "--expt-relaxed-constexpr"]
    others = [os.path.join(CSRC, f) for f in ("ctx.o", "eval.o", "kernels.o", "select.o", "eval_kernels.o")]
    procs = []
    for k in PROBES:
        obj = os.path.join(lib_dir, f"gemm_probe{k}.o")
        procs.append((k, obj, subprocess.Popen([NVCC, *flags, f"-DNPAIR_GRAD_PROBE={k}", "-c", os.path.join(CSRC, "gemm.cu"), "-o", obj])))
    for k, obj, pr in procs:
        if pr.wait():
            raise SystemExit(f"probe {k}: nvcc failed")
        subprocess.check_call([NVCC, *arch, "-shared", "-cudart", "static", "-o", os.path.join(lib_dir, f"libnpair_probe{k}.so"),
                               obj, *others, "-ldl"])


def run_one(precision, steps, warmup):
    """Child process: median gradient-phase milliseconds of the HL step with the library NPAIR_LIB points at."""
    import torch
    from npairloss_b200 import capi, synth
    from bench_retrieval_eval import PRECS
    c = synth.CONFIGS["HL"]
    B, D = c["B"], c["D"]
    x, lab = synth.make_inputs(B, D, 20171225 + c["idx"], noise=c["noise"])
    ctx = capi.Context(capi.make_config(B, D, sim_precision=PRECS[precision], **c["mining"]))
    dx, dl = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    grad = torch.empty_like(dx)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        ctx.forward(dx, dl)
        ctx.backward(1.0, grad)
    ctx.profile_enable(True)
    ms = []
    for _ in range(steps):
        flush.fill_(1)
        ctx.forward(dx, dl)
        ctx.backward(1.0, grad)
        ms.append(ctx.profile_read()[6])
    ctx.profile_enable(False)
    ctx.close()
    return statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build", action="store_true")
    ap.add_argument("--lib-dir", default=os.path.join(tempfile.gettempdir(), "npair_grad_probes"))
    ap.add_argument("--precisions", nargs="+", default=["fp16x2"], choices=["fp16x2", "bf16x3", "bf16"])
    ap.add_argument("--probes", nargs="+", type=int, default=sorted(PROBES), choices=sorted(PROBES))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps({"ms": run_one(args.child, args.steps, args.warmup)}))
        return
    if args.build:
        build(args.lib_dir)
        return
    from bench_retrieval_eval import ClockSampler, card
    for prec in args.precisions:
        for k in args.probes:
            env = dict(os.environ, NPAIR_LIB=os.path.join(args.lib_dir, f"libnpair_probe{k}.so"))
            with ClockSampler() as clk:
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", prec, "--steps", str(args.steps),
                                      "--warmup", str(args.warmup)], env=env, capture_output=True, text=True)
            if out.returncode:
                print(json.dumps({"precision": prec, "probe": PROBES[k], "error": out.stderr.strip().splitlines()[-1:]}))
                continue
            ms = json.loads(out.stdout.strip().splitlines()[-1])["ms"]
            print(json.dumps({"precision": prec, "probe": PROBES[k], "grad_gemm_ms": round(ms, 4), "card": card(),
                              "sm_clock_mhz_median": clk.median()}))


if __name__ == "__main__":
    main()
