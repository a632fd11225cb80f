"""Two real GPUs, NCCL: each sharded run equals the single-GPU run bit for bit in fitness and to fp32 (or fp64)
summation order in the update — the NES tape generation, CMA-ES on a sphere, closed-loop NES and CMA-ES, host-stepped
SynthWalk-v0 and mirrored sampling.  The ranks run through tests/ranks.spawn (a file store, no TCP port; killed after
its timeout).  Skipped on a one-GPU box (the CPU gloo tests cover the host logic there)."""
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import nes_oracle as orc
from ranks import spawn

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')]


def _tape_engine(N, precision, **kw):
    from distributedes_b200.engine import NESEngine
    d0, H, A, T = 24, 64, 4, 256
    obs, target = orc.synthetic_tape(T, d0, A)
    return NESEngine(state_dim=d0, hidden=H, action_dim=A, pop_size=N, theta0=orc.synthetic_theta(d0, H, A), obs=obs,
                     target=target, sigma=0.1, learning_rate=0.1, clip=1.0, seed=21, precision=precision, **kw)


def _tape(N, precision, use_graph, gens, comm):
    os.environ['DES_COMM'] = comm           # 'peer': kernels of this library over NVLink peer memory; 'nccl': two all-reduces
    eng = _tape_engine(N, precision, use_graph=use_graph)
    fit0 = theta1 = None
    for g in range(gens):
        eng.generation()
        if g == 0:
            fit0 = eng.fitness_all.cpu().numpy()
            theta1 = eng.theta.cpu().numpy()
    torch.cuda.synchronize()
    assert (eng.comm is not None) == (comm == 'peer'), 'exchange path %r was requested' % comm
    return dict(theta=eng.theta.cpu().numpy(), fitness=fit0, theta1=theta1)


@pytest.mark.parametrize('N,precision,use_graph,comm', [(1000, 'f16x3', False, 'peer'), (1001, 'fp32', False, 'nccl'),
                                                        (4096, 'f16', True, 'peer'), (1001, 'fp32', True, 'peer')])
def test_two_gpu_generation_matches_one_gpu(N, precision, use_graph, comm):
    r = spawn(2, _tape, N, precision, use_graph, 3, comm, backend='nccl')
    assert np.array_equal(r[0]['theta'], r[1]['theta'])            # identical parameters on both ranks, no broadcast
    assert np.array_equal(r[0]['fitness'], r[1]['fitness'])
    one = _tape_engine(N, precision, device='cuda:0')
    one.generation()
    # generation-0 fitness of a member does not depend on the sharding: bit-identical
    assert np.array_equal(one.fitness_all.cpu().numpy(), r[0]['fitness'])
    # the first update differs only by the order of the cross-shard fp32 sum.  (Later generations are not compared:
    # parameters that differ in the last bit flip near-tied ranks, which moves the update by ~5/N^1.5 per flip.)
    th0 = orc.synthetic_theta(24, 64, 4)
    th1 = one.theta.cpu().numpy()
    assert np.linalg.norm(th1 - r[0]['theta1']) <= 1e-5 * np.linalg.norm(th1 - th0)


def _cma_sphere():
    from distributedes_b200.cma_es import CMAEvolutionStrategy
    n, lam = 512, 130                                   # ragged shards
    es = CMAEvolutionStrategy(np.random.RandomState(0).randn(n), 1.0, lam, seed=6)
    X = es.ask()
    cost = es.gather_cost((X.double() ** 2).sum(1).float())
    es.tell(X, cost)
    torch.cuda.synchronize()
    return dict(C=es.C.cpu().numpy(), m=es.m.cpu().numpy(), sigma=es.sigma, X=X.cpu().numpy(), cost=cost.cpu().numpy())


def test_two_gpu_cma_generation_matches_one_gpu():
    """cma_es.CMAEvolutionStrategy sharded over 2 GPUs (all-reduce of the [n,n] rank-mu partials) against the same
    generation on one GPU: generation 0 has B = I, so both sample identical solutions from the counter noise."""
    from distributedes_b200.cma_es import CMAEvolutionStrategy
    r = spawn(2, _cma_sphere, backend='nccl')
    for k in ('C', 'm', 'sigma', 'cost'):
        assert np.array_equal(r[0][k], r[1][k]), k
    n, lam = 512, 130
    one = CMAEvolutionStrategy(np.random.RandomState(0).randn(n), 1.0, lam, seed=6, device='cuda:0')
    X = one.ask()
    assert np.array_equal(X.cpu().numpy(), np.concatenate([r[0]['X'], r[1]['X']]))
    cost = (X.double() ** 2).sum(1).float()
    one.tell(X, cost)
    C1 = one.C.cpu().numpy()
    assert np.linalg.norm(C1 - r[0]['C']) <= 1e-6 * np.linalg.norm(C1)          # order of the cross-shard fp32 sum
    assert np.linalg.norm(one.m.cpu().numpy() - r[0]['m']) <= 1e-12 * np.linalg.norm(r[0]['m'])


def _closed_loop():
    from distributedes_b200.engine import RolloutEngine
    eng = RolloutEngine(hidden=64, pop_size=37, theta0=orc.synthetic_theta(3, 64, 1), sigma=0.1, learning_rate=0.1, seed=3)
    eng.generation()
    fit0, stats0 = eng.fitness_all.cpu().numpy().copy(), eng.obs_stats.cpu().numpy().copy()
    eng.generation()
    return dict(theta=eng.theta_numpy(), stats=eng.obs_stats.cpu().numpy(), fit=eng.fitness_all.cpu().numpy(),
                fit0=fit0, stats0=stats0)


def test_two_gpu_closed_loop_equals_one_gpu():
    from distributedes_b200.engine import RolloutEngine
    r0, r1 = spawn(2, _closed_loop, backend='nccl')
    for k in ('theta', 'stats', 'fit'):
        assert np.array_equal(r0[k], r1[k]), k
    eng = RolloutEngine(hidden=64, pop_size=37, theta0=orc.synthetic_theta(3, 64, 1), sigma=0.1, learning_rate=0.1, seed=3)
    eng.generation()
    assert np.array_equal(eng.fitness_all.cpu().numpy(), r0['fit0'])
    assert np.allclose(eng.obs_stats.cpu().numpy(), r0['stats0'], rtol=1e-6)


def _closed_loop_cma():
    """Three generations of closed-loop CMA-ES (Pendulum-v0, 16 hidden units, lambda = 37: a ragged 19 + 18 split)."""
    from distributedes_b200 import cma_es
    from distributedes_b200.config import ClosedLoopPendulumConfig
    cfg = ClosedLoopPendulumConfig(16)
    cfg.pop_size, cfg.sigma, cfg.seed, cfg.max_generations = 37, 0.5, 3, 3
    worker = cma_es.Worker(0, None, None, None, None, cfg)
    es = cma_es.CMAEvolutionStrategy(cfg.initial_weight, cfg.sigma, cfg.pop_size, seed=cfg.seed, device=worker.device)
    costs = []
    real_run = worker.run

    def spy_run(solutions, member_offset=0, generation=0):
        cost = real_run(solutions, member_offset, generation)
        costs.append(es.gather_cost(cost).cpu().numpy().copy())
        return cost
    worker.run = spy_run
    rewards, _, _ = cma_es.train(cfg, worker=worker, es=es)
    return dict(cost=np.stack(costs), stats=worker.obs_stats.cpu().numpy(), m=es.m.cpu().numpy(),
                rewards=np.asarray(rewards))


def test_two_gpu_closed_loop_cma_equals_one_gpu():
    r0, r1 = spawn(2, _closed_loop_cma, backend='nccl')
    for k in ('cost', 'stats', 'm', 'rewards'):
        assert np.array_equal(r0[k], r1[k]), k
    one = _closed_loop_cma()
    assert np.array_equal(one['cost'][0], r0['cost'][0])      # per-member fitness is shard invariant
    # the observation totals and sum_i w_i y_i are summed per rank, then across ranks: fp64 association differs
    assert np.allclose(one['stats'], r0['stats'], rtol=1e-6, atol=1e-7)
    assert np.allclose(one['m'], r0['m'], rtol=1e-9, atol=1e-9)


def _host_env(comm=None):
    """HostEnvEngine on SynthWalk-v0, each rank stepping only its own members' environments."""
    from distributedes_b200.engine import HostEnvEngine
    from distributedes_b200.envs import GymEnvBatch
    from oracle import synth_walk as sw
    if comm is not None:
        os.environ.setdefault('DES_COMM', comm)
    eng = HostEnvEngine(env_fn=sw.SynthWalkEnv, batch_env_fn=lambda B: GymEnvBatch(sw.SynthWalkEnv, B, 4), hidden=64,
                        pop_size=13, theta0=orc.synthetic_theta(24, 64, 4), sigma=0.1, learning_rate=0.1,
                        repetitions=4, seed=4)
    fit, steps = [], []
    for _ in range(2):
        eng.generation()
        fit.append(eng.fitness_all.cpu().numpy().copy())
        steps.append(eng.steps_taken)
    torch.cuda.synchronize()
    return dict(fit=np.stack(fit), steps=np.asarray(steps), stats=eng.obs_stats.cpu().numpy(), theta=eng.theta_numpy())


def test_two_gpu_host_env_equals_one_gpu():
    r0, r1 = spawn(2, _host_env, 'nccl', backend='nccl')
    for k in ('fit', 'steps', 'stats', 'theta'):
        assert np.array_equal(r0[k], r1[k]), k
    one = _host_env()
    assert np.array_equal(one['fit'], r0['fit']) and np.array_equal(one['steps'], r0['steps'])
    assert np.allclose(one['stats'], r0['stats'], rtol=1e-6, atol=1e-7)


def _mirrored():
    from distributedes_b200.engine import NESEngine
    d0, H, A, T = 24, 64, 4, 256
    obs, target = orc.synthetic_tape(T, d0, A)
    eng = NESEngine(state_dim=d0, hidden=H, action_dim=A, pop_size=22, theta0=orc.synthetic_theta(d0, H, A), obs=obs,
                    target=target, sigma=0.1, learning_rate=0.05, seed=3, precision='f16x3', mirrored=True)
    for _ in range(2):
        eng.generation()
    return dict(theta=eng.theta_numpy(), fit=eng.fitness_all.cpu().numpy(), offset=eng.offset, n_local=eng.n_local)


def test_two_gpu_mirrored_equals_one_gpu():
    r = spawn(2, _mirrored, backend='nccl')
    assert (int(r[0]['n_local']), int(r[1]['offset'])) == (12, 12)
    assert np.array_equal(r[0]['theta'], r[1]['theta']) and np.array_equal(r[0]['fit'], r[1]['fit'])
    one = _mirrored()
    assert np.array_equal(one['fit'], r[0]['fit'])
    assert np.max(np.abs(one['theta'] - r[0]['theta'])) <= 1e-6
