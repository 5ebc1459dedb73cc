"""Developer probe: run one config through the handle API, print the LM trace and per-kernel CUDA-event timings."""
import json
import sys
import time

import numpy as np
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ccm_slam_b200 import api, synth

name = sys.argv[1] if len(sys.argv) > 1 else "cfg4"
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
api.init(0)
t = time.time(); p = synth.make_config(name); print(f"[{name}] generated K={p.K} P={p.P} E={p.E} in {time.time()-t:.1f}s", flush=True)
t = time.time(); h = api.BAHandle(p); print(f"create: {time.time()-t:.3f}s info={h.info()}", flush=True)
t = time.time(); r = h.optimize(iterations=iters, want_state=False); dt = time.time() - t
print(f"optimize({iters}): {dt:.3f}s iters={r['iters_done']} trials={r['trials_total']} pcg_total={r['pcg_iters_total']} notconv={r['pcg_not_converged']}")
print("trace [it lambda chi2 rho trials lambda_after pcg_it relres]"); np.set_printoptions(linewidth=200, precision=4)
print(r["trace"])
names = ["linearize", "pose_pass", "residual", "z_only", "schur", "backsub", "pcg"]
lam = float(r["trace"][0, 1]) if len(r["trace"]) else 1.0
for i, n in enumerate(names):
    print(f"  kernel {n:12s}: {h.time_kernel(i, reps=3, lam=lam):9.4f} ms")
print("launches", api.kernel_launches())
import ctypes as C
cyc = np.zeros(8, np.int64)
api.lib().ccm_ba_debug_pcg_cycles(h._h, cyc.ctypes.data_as(C.c_void_p))
if cyc.sum() > 0:
    names = ["setup", "spmv", "update+restrict", "coarse", "precond", "unused", "-", "-"]
    print("pcg phase cycles (CTA 0):", {n: int(c) for n, c in zip(names, cyc)}, "share:", {n: round(float(c) / cyc.sum(), 3) for n, c in zip(names, cyc) if c})
