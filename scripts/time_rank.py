"""Time des_centered_rank (CUDA events).  python scripts/time_rank.py"""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from distributedes_b200 import ops
res = []
flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
# N <= 2048 takes the counting rank, larger populations the bucketed one
for N, n in [(256, 256), (2048, 2048), (2048, 1024), (65536, 65536), (65536, 8192), (16384, 16384), (16384, 8192), (4096, 4096),
             (262144, 262144)]:
    f = torch.randn(N, device='cuda')
    ws = ops.rank_workspace(n, 'cuda', N); out = torch.empty(n, device='cuda')
    for _ in range(3): ops.centered_rank(f, 0, n, workspace=ws, out=out)
    reps = 20
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps): ops.centered_rank(f, 0, n, workspace=ws, out=out)
    ev[1].record(); torch.cuda.synchronize()
    warm = ev[0].elapsed_time(ev[1]) / reps
    cold = []
    for _ in range(5):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); ops.centered_rank(f, 0, n, workspace=ws, out=out); b.record(); torch.cuda.synchronize()
        cold.append(a.elapsed_time(b))
    res.append(dict(N=N, n_local=n, warm_us=round(warm * 1e3, 1), cold_us=round(min(cold) * 1e3, 1)))
print(json.dumps(res))
