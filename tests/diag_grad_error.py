"""Diagnostic (not a test): gradient / loss error of the CUDA path against the oracle (on the GPU's own S) as the database grows.
   python tests/diag_grad_error.py [D] [B,B,...] [grad_chunk_cols] [usage,rand,hard,c3] [synth | cone epsilon, e.g. 0.02]
   Cone inputs (grad_ref.cone_inputs) are unit rows of pairwise cosine ~1 / (1 + epsilon^2), where a row's weights are nearly equal."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from npairloss_b200 import capi, synth
from oracle import oracle_lib as o
from gpu_harness import gpu_step_world
from grad_ref import cone_inputs
D = int(sys.argv[1]) if len(sys.argv) > 1 else 512
chunk = int(sys.argv[3]) if len(sys.argv) > 3 else 0
minings = {"usage": synth.USAGE_MINING, "rand": synth.DEFAULT_MINING, "hard": dict(synth.DEFAULT_MINING, ap_method=0, an_method=0),
           "c3": dict(synth.DEFAULT_MINING, an_method=0)}
mnames = sys.argv[4].split(",") if len(sys.argv) > 4 else ["usage"]
Bs = [int(b) for b in sys.argv[2].split(",")] if len(sys.argv) > 2 else [1024, 2048, 4096, 8192]
inputs = sys.argv[5] if len(sys.argv) > 5 else "synth"
for B in Bs:
    x, lab = synth.make_inputs(B, D, 20171225 + 5, noise=2.5) if inputs == "synth" else cone_inputs(B, D, float(inputs), 20171225 + 5)
    for mname in mnames:
        prec, name, mining = 2, "fp16x2 " + mname, minings[mname]
        g = gpu_step_world(x, lab, B, 1, mining, prec, capi.GEMM_TCGEN05, grad_chunk_cols=chunk)
        t0 = time.time()
        cfg = o.make_config(B, D, faithful_sorts=0, **mining)
        tops_o, dx_o = o.step_world(x, lab, cfg, 1.0, S_inject_all=g["S"])
        rel = np.linalg.norm(g["dx"] - dx_o) / np.linalg.norm(dx_o)
        proj = float((g["dx"].astype(np.float64) * dx_o).sum() / (dx_o.astype(np.float64) ** 2).sum())
        print(f"B={B} D={D} {inputs} {name}: loss_rel={abs(g['tops'][0,0]-tops_o[0,0])/abs(tops_o[0,0]):.2e} grad_rel={rel:.2e} shrink={proj-1:+.2e} "
              f"tops_gpu={g['tops'][0,1:4]} tops_o={tops_o[0,1:4]} oracle_s={time.time()-t0:.1f}", flush=True)
