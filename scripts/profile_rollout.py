"""Two closed-loop generations at the given population for a profiler (argv: pop hidden)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from distributedes_b200.engine import RolloutEngine
from distributedes_b200.model import StandardFCNet
N, H = int(sys.argv[1]), int(sys.argv[2])
eng = RolloutEngine(hidden=H, pop_size=N, theta0=StandardFCNet(3, 1, H, seed=0).get_weight(), sigma=0.1, learning_rate=0.1, seed=1)
for _ in range(2):
    eng.generation()
torch.cuda.synchronize()
