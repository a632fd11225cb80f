"""Time the CMA rank-mu kernels (BASELINE configs[2] and [4] shapes, and both sides of ops.CMA_TC_MIN_N) with CUDA events."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from distributedes_b200 import ops
out = []
for n, lam in [(1024, 256), (2047, 256), (2048, 256), (4096, 1024), (4096, 128)]:   # FFMA below n = 2048, tensor cores from it
    Y = torch.randn(lam, n, device='cuda'); w = torch.rand(lam, device='cuda'); C = torch.eye(n, device='cuda'); pc = torch.randn(n, device='cuda')
    dC = ops.cma_rank_mu(Y, w)
    for _ in range(3):
        ops.cma_rank_mu(Y, w, out=dC); ops.cma_cov_apply(C, dC, pc, decay=0.99, c1=0.001, cmu=0.009)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    reps = 20
    ev[0].record()
    for _ in range(reps): ops.cma_rank_mu(Y, w, out=dC)
    ev[1].record()
    for _ in range(reps): ops.cma_cov_apply(C, dC, pc, decay=0.99, c1=0.001, cmu=0.009)
    ev[2].record(); torch.cuda.synchronize()
    t1 = ev[0].elapsed_time(ev[1]) / reps; t2 = ev[1].elapsed_time(ev[2]) / reps
    out.append(dict(n=n, lam=lam, rank_mu_ms=t1, rank_mu_tflops=2 * lam * n * n / t1 / 1e9, cov_apply_ms=t2,
                    cov_apply_gbs=12 * n * n / t2 / 1e6))
print(json.dumps(out))
