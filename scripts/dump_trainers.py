#!/usr/bin/env python
"""Seeded outputs of every NES and CMA-ES mode, through the public constructors and train() functions only, into one
.npz: theta, fitness, observation statistics, test returns and step counts.  Two builds run with the same arguments can
be compared file for file (the outputs are deterministic).

    python scripts/dump_trainers.py OUT.npz [--gens 3]
"""
import argparse
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import nes_oracle as orc  # noqa: E402
from oracle import synth_walk as sw  # noqa: E402


class Cfg:
    """The attributes natural_es.train reads."""

    def __init__(self, d0, gens, reps=1, test_reps=1):
        self.state_dim, self.pop_size, self.repetitions, self.test_repetitions = d0, 0, reps, test_reps
        self.max_steps, self.max_generations = 0, gens


def nes_engines():
    from distributedes_b200.engine import HostEnvEngine, NESEngine, RolloutEngine
    from distributedes_b200.envs import GymEnvBatch
    d0, H, A, T = 24, 64, 4, 256
    obs, target = orc.synthetic_tape(T, d0, A)
    for prec in ('fp32', 'f16x3', 'f16'):
        for mirrored in (False, True):
            for norm in (False, True):
                def tape(use_graph, prec=prec, mirrored=mirrored, norm=norm):
                    return NESEngine(state_dim=d0, hidden=H, action_dim=A, pop_size=1024, theta0=orc.synthetic_theta(d0, H, A),
                                     obs=obs, target=target, sigma=0.1, learning_rate=0.05, seed=3, precision=prec,
                                     normalize_obs=norm, repetitions=2 if norm else 1, mirrored=mirrored,
                                     use_graph=use_graph)
                yield 'tape_%s_m%d_n%d' % (prec, mirrored, norm), tape, Cfg(d0, 0, 2 if norm else 1, 2)
    for mirrored in (False, True):
        def rollout(use_graph, mirrored=mirrored):
            return RolloutEngine(hidden=64, pop_size=512, theta0=orc.synthetic_theta(3, 64, 1, seed=2), sigma=0.1,
                                 learning_rate=0.05, seed=5, repetitions=10, action_noise_std=0.1, mirrored=mirrored,
                                 use_graph=use_graph)
        yield 'device_m%d' % mirrored, rollout, Cfg(3, 0, 10, 10)

        def host(use_graph, mirrored=mirrored):
            return HostEnvEngine(env_fn=sw.SynthWalkEnv, batch_env_fn=lambda B: GymEnvBatch(sw.SynthWalkEnv, B, 4),
                                 hidden=16, pop_size=24, theta0=np.asarray(orc.synthetic_theta(24, 16, 4), np.float32),
                                 sigma=0.1, learning_rate=0.1, repetitions=3, test_repetitions=2, seed=4,
                                 mirrored=mirrored, use_graph=use_graph)
        yield 'host_m%d' % mirrored, host, Cfg(24, 0, 3, 2)


def cma_configs(gens):
    from distributedes_b200.config import BipedalWalkerConfig, ClosedLoopPendulumConfig, HostEnvConfig
    from distributedes_b200.envs import GymEnvBatch
    tape = BipedalWalkerConfig(hidden_size=16, tape_len=64)
    tape.pop_size, tape.sigma, tape.test_repetitions = 64, 1.0, 2
    device = ClosedLoopPendulumConfig(16)
    device.pop_size, device.sigma = 16, 1.0
    host = HostEnvConfig(sw.SynthWalkEnv, hidden_size=16, task='SynthWalk-v0',
                         batch_env_fn=lambda B: GymEnvBatch(sw.SynthWalkEnv, B, 6))
    host.pop_size, host.sigma, host.repetitions, host.test_repetitions = 12, 0.5, 3, 2
    for name, cfg in (('tape', tape), ('device', device), ('host', host)):
        cfg.seed, cfg.max_generations = 6, gens
        yield name, cfg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--gens', type=int, default=3)
    a = ap.parse_args()
    from distributedes_b200 import cma_es, natural_es
    out = {}
    for name, make, cfg in nes_engines():
        # natural_es.train: evaluate / rank / apply, test episodes and step counts
        eng = make(False)
        cfg.pop_size, cfg.max_generations = eng.N, a.gens
        rewards, steps, _ = natural_es.train(cfg, engine=eng)
        out['nes_%s_rewards' % name], out['nes_%s_steps' % name] = np.asarray(rewards), np.asarray(steps)
        out['nes_%s_theta' % name] = eng.theta_numpy()
        out['nes_%s_fitness' % name] = eng.fitness_all.cpu().numpy()
        if eng.normalize_obs:
            out['nes_%s_stats' % name] = eng.obs_stats.cpu().numpy()
        # generation(): the CUDA graph where the engine captures one
        eng = make(True)
        fits = []
        for _ in range(a.gens):
            eng.generation()
            fits.append(eng.fitness_all.cpu().numpy())
        out['nes_%s_gen_fitness' % name], out['nes_%s_gen_theta' % name] = np.stack(fits), eng.theta_numpy()
        print(name, flush=True)
    for name, cfg in cma_configs(a.gens):
        worker = cma_es.Worker(0, None, None, None, None, cfg)
        es = cma_es.CMAEvolutionStrategy(cfg.initial_weight, cfg.sigma, cfg.pop_size, seed=cfg.seed, device=worker.device)
        rewards, steps, _ = cma_es.train(cfg, worker=worker, es=es)
        out['cma_%s_rewards' % name], out['cma_%s_steps' % name] = np.asarray(rewards), np.asarray(steps)
        out['cma_%s_m' % name], out['cma_%s_C' % name] = es.m.cpu().numpy(), es.C.cpu().numpy()
        if getattr(worker, 'obs_stats', None) is not None:
            out['cma_%s_stats' % name] = worker.obs_stats.cpu().numpy()
        print('cma', name, flush=True)
    torch.cuda.synchronize()
    np.savez(a.out, **out)


if __name__ == '__main__':
    main()
