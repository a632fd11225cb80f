"""One rank's kernels of an 8-way sharded generation on ONE GPU (for a profiler launch list): members [0, 8192) of N = 65536.
python scripts/profile_shard.py [N] [n_local] [hidden] [gens]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from oracle import nes_oracle as orc
from distributedes_b200 import ops
N = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
n = int(sys.argv[2]) if len(sys.argv) > 2 else 8192
H = int(sys.argv[3]) if len(sys.argv) > 3 else 256
gens = int(sys.argv[4]) if len(sys.argv) > 4 else 3
d0, A, T = 24, 4, 256
dev = 'cuda:0'
obs, target = orc.synthetic_tape(T, d0, A)
th = torch.from_numpy(orc.synthetic_theta(d0, H, A)).to(dev)
o, t = torch.from_numpy(obs).to(dev), torch.from_numpy(target).to(dev)
P = th.numel()
fit = torch.randn(N, device=dev)
shaped = torch.zeros(n, device=dev)
partial = torch.zeros(P, device=dev)
m = torch.zeros(P, dtype=torch.float64, device=dev); v = torch.zeros_like(m)
upd = torch.zeros(P, device=dev)
st = ops.new_state(dev, 0)
rws = ops.rank_workspace(n, dev, N); gws = ops.grad_workspace(n, P, dev)
for g in range(gens):
    ops.nes_eval(th, o, t, hidden=H, sigma=0.1, clip=1.0, seed=0, state=st, member_offset=0, n_local=n, precision='f16x3', out=fit[:n])
    ops.centered_rank(fit, 0, n, workspace=rws, out=shaped)
    ops.nes_grad_partial(shaped, P, seed=0, state=st, member_offset=0, workspace=gws, out=partial)
    ops.nes_apply(th, m, v, partial, N, st, sigma=0.1, learning_rate=0.1, update_out=upd)
    ops.state_advance(st)
torch.cuda.synchronize()
print('done')
