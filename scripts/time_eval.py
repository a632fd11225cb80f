"""Time des_nes_eval (CUDA events) and check it against the fp32 CUDA-core path on a sample of members.
python scripts/time_eval.py [pop] [hidden] [precision] [reps] [check_members]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import json
import torch
from oracle import nes_oracle as orc
from distributedes_b200 import ops

pop = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
H = int(sys.argv[2]) if len(sys.argv) > 2 else 256
prec = sys.argv[3] if len(sys.argv) > 3 else 'f16x3'
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 5
ncheck = int(sys.argv[5]) if len(sys.argv) > 5 else 600
d0, A, T = 24, 4, 256
dev = 'cuda:0'
obs, target = orc.synthetic_tape(T, d0, A)
th = torch.from_numpy(orc.synthetic_theta(d0, H, A)).to(dev)
o, t = torch.from_numpy(obs).to(dev), torch.from_numpy(target).to(dev)
kw = dict(hidden=H, sigma=0.1, clip=1.0, seed=9, generation=2, member_offset=0)
out = {'pop': pop, 'H': H, 'precision': prec}
if ncheck:
    a = ops.nes_eval(th, o, t, precision='fp32', n_local=ncheck, **kw)
    b = ops.nes_eval(th, o, t, precision=prec, n_local=ncheck, **kw)
    torch.cuda.synchronize()
    out['max_rel_vs_fp32'] = float(((a - b).abs() / a.abs()).max())
    b2 = ops.nes_eval(th, o, t, precision=prec, n_local=ncheck, **kw)
    out['deterministic'] = bool(torch.equal(b, b2))
    ref = orc.evaluate_population(th.cpu().numpy(), obs, target, 0.1, 1.0, 9, 2, 0, 8, d0, H, A)
    out['max_rel_vs_oracle8'] = float(abs((b[:8].cpu().numpy() - ref) / ref).max())
for _ in range(2):
    f = ops.nes_eval(th, o, t, precision=prec, n_local=pop, **kw)
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
ev[0].record()
for i in range(reps):
    f = ops.nes_eval(th, o, t, precision=prec, n_local=pop, **kw)
    ev[i + 1].record()
torch.cuda.synchronize()
ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]
out['ms'] = [round(x, 3) for x in ms]
out['ms_min'] = round(min(ms), 3)
out['fit_mean'] = float(f.mean())
print(json.dumps(out))
