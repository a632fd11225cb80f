"""Run a few eager NES generations (for a profiler: torch.profiler or CUDA events around the kernels).  python scripts/profile_gen.py [pop] [hidden] [precision] [gens]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from oracle import nes_oracle as orc
from distributedes_b200.engine import NESEngine
pop = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
H = int(sys.argv[2]) if len(sys.argv) > 2 else 256
prec = sys.argv[3] if len(sys.argv) > 3 else 'f16'
gens = int(sys.argv[4]) if len(sys.argv) > 4 else 3
d0, A, T = 24, 4, 256
obs, target = orc.synthetic_tape(T, d0, A)
eng = NESEngine(state_dim=d0, hidden=H, action_dim=A, pop_size=pop, theta0=orc.synthetic_theta(d0, H, A), obs=obs,
                target=target, sigma=0.1, learning_rate=0.1, clip=1.0, seed=0, precision=prec, device='cuda:0')
for _ in range(gens):
    eng.generation()
torch.cuda.synchronize()
print('done', float(eng.fitness_all.mean()))
