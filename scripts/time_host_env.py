#!/usr/bin/env python
"""Timing of the host-stepped path (DESIGN §4.8, §8): des_policy_act per step against the bytes it must read, the
bridge's whole step with a no-op vectorised environment, and a host-stepped Pendulum-v0 generation next to
des_rollout_eval's.

    python scripts/time_host_env.py [--out results.json]

Shapes: H = 64, d0 = 24, A = 4, 10 repetitions (BipedalWalker with the reference's NES width); n_local in {64, 1024,
16384}.  The kernel is timed with CUDA events over many launches; the step with the host clock after a synchronise."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributedes_b200 import ops                       # noqa: E402
from distributedes_b200.fitness import HostEpisodes       # noqa: E402
from oracle import nes_oracle as orc                     # noqa: E402
from oracle import pendulum_oracle as po                 # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # H100 SXM5 80 GB HBM3 peak


class NoopEnv:
    """Vectorised environment that costs nothing: zero observations, every episode `length` steps."""

    def __init__(self, B, d0, length):
        self.num_envs, self.d0, self.length = B, d0, length

    def reset(self, keys):
        self.t = 0
        return np.zeros((self.num_envs, self.d0))

    def step(self, actions, alive):
        self.t += 1
        return np.zeros((self.num_envs, self.d0)), np.zeros(self.num_envs), np.full(self.num_envs, self.t >= self.length)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'not reported'
    return name, pl or 'not reported'


def time_kernel(n, d0=24, H=64, A=4, reps=10, iters=200):
    P = orc.param_count(d0, H, A)
    rows = torch.randn(n, P, device='cuda') * 0.1
    obs = torch.randn(n, reps, d0, device='cuda')
    alive = torch.ones(n, reps, dtype=torch.uint8, device='cuda')
    stats = torch.cat([torch.zeros(d0), torch.ones(d0), torch.tensor([100.0])]).cuda()
    part = torch.zeros(n, 2 * d0 + 1, dtype=torch.float64, device='cuda')
    out = torch.empty(n, reps, A, device='cuda')
    kw = dict(state_dim=d0, hidden=H, action_dim=A, repetitions=reps, clip=1.0, seed=1, generation=0, obs_stats=stats,
              stat_part=part, out=out)
    for t in range(10):
        ops.policy_act(rows, obs, alive, t=t, **kw)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for t in range(iters):
        ops.policy_act(rows, obs, alive, t=t, **kw)
    e.record()
    torch.cuda.synchronize()
    us = s.elapsed_time(e) * 1e3 / iters
    nbytes = n * P * 4
    return dict(n_local=n, P=P, kernel_us=us, bytes=nbytes, hbm_bound_us=nbytes / HBM_BYTES_PER_S * 1e6,
                achieved_GBps=nbytes / (us * 1e-6) / 1e9)


def time_bridge(n, d0=24, H=64, A=4, reps=10, length=100):
    P = orc.param_count(d0, H, A)
    rows = torch.randn(n, P, device='cuda') * 0.1
    ep = HostEpisodes(ops, 'cuda', NoopEnv(n * reps, d0, length), n, reps, d0, H, A, 1.0, 0.0, 1)
    stats = torch.zeros(2 * d0 + 1, device='cuda')
    part = torch.zeros(n, 2 * d0 + 1, dtype=torch.float64, device='cuda')
    ep.run(rows, generation=0, obs_stats=stats, stat_part=part)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ep.run(rows, generation=1, obs_stats=stats, stat_part=part)
    torch.cuda.synchronize()
    return dict(n_local=n, step_us=(time.perf_counter() - t0) / length * 1e6)


def time_pendulum(N, H=64, reps=10):
    theta = torch.from_numpy(orc.synthetic_theta(3, H, 1)).cuda()
    stats = torch.cat([torch.zeros(3), torch.ones(3), torch.tensor([100.0])]).cuda()
    rows = torch.empty(N, orc.param_count(3, H, 1), device='cuda')
    ep = HostEpisodes(ops, 'cuda', po.PendulumBatch(N * reps, 3), N, reps, 3, H, 1, 2.0, 0.0, 3)
    part = torch.zeros(N, 7, dtype=torch.float64, device='cuda')
    res = {}
    for name in ('host', 'device'):
        for rep in range(2):                                   # the first run warms up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if name == 'host':
                ops.nes_perturb(theta, N, 0.1, 3, rep, out=rows)
                ep.run(rows, generation=rep, obs_stats=stats, stat_part=part)
            else:
                ops.rollout_eval(theta, hidden=H, repetitions=reps, sigma=0.1, clip=2.0, seed=3, generation=rep,
                                 n_local=N, obs_stats=stats)
            torch.cuda.synchronize()
            res[name + '_ms'] = (time.perf_counter() - t0) * 1e3
    res['N'] = N
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, pl = card()
    res = dict(card=name, power_limit=pl, kernel=[time_kernel(n) for n in (64, 1024, 16384)],
               bridge=[time_bridge(n, length=100 if n < 16384 else 20) for n in (64, 1024, 16384)],
               pendulum=[time_pendulum(N) for N in (64, 4096)])
    print('%s, power limit %s' % (name, pl))
    for k in res['kernel']:
        print('policy_act n_local=%5d  %8.1f us/step  (%.1f MB of weights: HBM bound %.1f us, %.0f GB/s achieved)'
              % (k['n_local'], k['kernel_us'], k['bytes'] / 1e6, k['hbm_bound_us'], k['achieved_GBps']))
    for b in res['bridge']:
        print('whole step, no-op env n_local=%5d  %8.1f us' % (b['n_local'], b['step_us']))
    for p in res['pendulum']:
        print('Pendulum generation N=%4d x 10 x 200: host-stepped %.1f ms, des_rollout_eval %.2f ms'
              % (p['N'], p['host_ms'], p['device_ms']))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
