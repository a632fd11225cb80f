"""Time R independent NES runs of 64 members on the closed-loop Pendulum two ways: R RolloutEngine runs one after another
against one RolloutRunsEngine of R runs.  H in {16, 64}, 10 x 200-step episodes per member, R in {1, 4, 10, 32}.

  generation   ms per generation of all R runs, from CUDA events around `iters` generations after a warm-up, with the L2
               flushed before each timed window (the sequential arm times each run's generations and sums them)
  train        seconds of natural_es.train run R times against natural_es.train_runs(config, R), 5 generations each,
               test episodes included, from a host clock around work that ends in a device synchronise

Prints one JSON line with the card's name and power limit, read in the same call.

    python scripts/time_runs.py [--iters 20] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributedes_b200 import config as cfg          # noqa: E402
from distributedes_b200 import natural_es             # noqa: E402
from distributedes_b200.engine import RolloutEngine, RolloutRunsEngine   # noqa: E402
from distributedes_b200.model import StandardFCNet    # noqa: E402

POP = 64
_L2 = None


def flush_l2():
    global _L2
    if _L2 is None:
        _L2 = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')      # > the H100's 50 MB L2
    _L2.zero_()


def timed(fn, iters):
    """ms per call of fn over `iters` calls, CUDA events, L2 flushed before the window."""
    flush_l2()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def generation_ms(H, R, iters):
    theta0 = StandardFCNet(3, 1, H, seed=0).get_weight()
    kw = dict(hidden=H, pop_size=POP, theta0=theta0, sigma=0.1, learning_rate=0.1, seed=1)
    singles = [RolloutEngine(use_graph=True, **kw) for _ in range(R)]
    batch = RolloutRunsEngine(runs=R, use_graph=True, **kw)
    for _ in range(3):                                   # warm-up: graph capture, module loading
        batch.generation()
        for e in singles:
            e.generation()
    torch.cuda.synchronize()
    seq = sum(timed(e.generation, iters) for e in singles)
    bat = timed(batch.generation, iters)
    return seq, bat


def train_s(H, R):
    c = cfg.ClosedLoopPendulumConfig(H)
    c.pop_size, c.max_generations = POP, 4               # 5 evaluations and test collections
    natural_es.train(c)                                  # warm-up
    natural_es.train_runs(c, R)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(R):
        natural_es.train(c)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    natural_es.train_runs(c, R)
    torch.cuda.synchronize()
    return t1 - t0, time.perf_counter() - t1


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_runs.py measures on a GPU; none is available')
    torch.cuda.set_device(0)
    rows = []
    for H in (16, 64):
        for R in (1, 4, 10, 32):
            seq, bat = generation_ms(H, R, a.iters)
            tseq, tbat = train_s(H, R)
            rows.append(dict(hidden=H, runs=R, pop=POP, seq_generation_ms=round(seq, 4), batch_generation_ms=round(bat, 4),
                             generation_speedup=round(seq / bat, 2), seq_train_s=round(tseq, 3),
                             batch_train_s=round(tbat, 3), train_speedup=round(tseq / tbat, 2)))
            print(json.dumps(rows[-1]), file=sys.stderr)
    res = dict(card=card(), results=rows)
    print(json.dumps(res))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
