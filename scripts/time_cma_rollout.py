"""Time closed-loop CMA-ES generations on Pendulum-v0 (10 x 200-step episodes per solution) with CUDA events, split into
ask() (z + sampling GEMM), rollouts (des_rollout_eval_solutions), tell() without the eigendecomposition (rank shaping,
rank-mu, covariance update) and the eigendecomposition itself (its lazy refresh: every 13 generations at H = 64 and
lambda = 64, every generation at lambda >= 4096).  Each shape is timed over enough generations to cover one refresh and
reported as the per-generation mean, with the card's name and power limit read in the same run.

    python scripts/time_cma_rollout.py
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np      # noqa: E402
import torch            # noqa: E402
from distributedes_b200 import cma_es, ops          # noqa: E402
from distributedes_b200.config import ClosedLoopPendulumConfig       # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = 'nvidia-smi unavailable (%s)' % e
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q)


def time_shape(H, lam, reps=10, warmup=1):
    cfg = ClosedLoopPendulumConfig(H)
    cfg.pop_size, cfg.sigma, cfg.repetitions = lam, 0.5, reps
    worker = cma_es.Worker(0, None, None, None, None, cfg)
    es = cma_es.CMAEvolutionStrategy(cfg.initial_weight, cfg.sigma, lam, seed=1, device=worker.device)
    gap = es.eigen_gap
    es.eigen_gap = 1 << 30                     # the refresh is run and timed below, where tell() would run it
    gens = max(gap, 3)
    phases = dict(ask=0.0, rollout=0.0, tell=0.0, eigh=0.0)
    for g in range(warmup + gens):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        ev[0].record()
        X = es.ask()
        ev[1].record()
        cost = worker.run(X, es.offset, es.gen)
        ev[2].record()
        shaped = ops.centered_rank(cost.contiguous())
        es.tell(X, shaped)
        worker.merge_obs_stats(es)
        ev[3].record()
        if es.gen % gap == 0:
            d2, es.B = torch.linalg.eigh(es.C.to(torch.float64))
            es.D = torch.sqrt(torch.clamp(d2, min=1e-300))
        ev[4].record()
        torch.cuda.synchronize()
        if g >= warmup:
            for k, name in enumerate(('ask', 'rollout', 'tell', 'eigh')):
                phases[name] += ev[k].elapsed_time(ev[k + 1]) / gens
    total = sum(phases.values())
    return dict(hidden=H, n=es.n, lam=lam, reps=reps, eigen_gap=gap, generations=gens,
                **{k + '_ms': round(v, 3) for k, v in phases.items()}, generation_ms=round(total, 3),
                env_steps_per_s=round(lam * reps * 200 / total * 1e3))


if __name__ == '__main__':
    torch.cuda.set_device(0)
    print(json.dumps(dict(card=card())))
    for H in (16, 64):
        for lam in (64, 4096, 16384):
            print(json.dumps(time_shape(H, lam)), flush=True)
