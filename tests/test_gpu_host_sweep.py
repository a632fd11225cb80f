"""Host-stepped sweeps on the GPU.  Each sweep entry point is bit-equal, run by run, to the single entry point with run
r's seed, sigma and action noise at member_offset 0: the weight rows, the policy step (every policy width, state_dim up to
32, action_dim up to 8, repetitions up to 16, statistics on and off, action noise on and off, dead slots, a NaN
observation of an alive slot, run_size 1 for the test episodes) and the per-run observation totals.
HostEnvSweepEngine is R HostEnvEngines bit for bit, and train_sweep with the train_host_walk golden config as one of
its runs gives train()'s rewards and steps for every run."""
import copy
import os

import numpy as np
import pytest
import torch

from distributedes_b200.fitness import POLICY_WIDTHS
from oracle import nes_oracle as orc
from oracle import synth_walk as sw

pytestmark = pytest.mark.gpu


def _hyper(R, rng, noise=True):
    """Per-run seeds (two runs share one), sigma, learning rate, weight decay and action noise."""
    seeds = [int(s) for s in rng.integers(0, 2**63, R)]
    if R > 2:
        seeds[2] = seeds[0]
    return dict(seeds=seeds, sigma=list(rng.uniform(0.02, 0.3, R)), learning_rate=list(rng.uniform(0.01, 0.2, R)),
                weight_decay=list(rng.uniform(0.0, 0.02, R)),
                action_noise_std=list(rng.uniform(0.1, 0.5, R)) if noise else [0.0] * R)


def _table(h):
    from distributedes_b200 import ops_sweep
    return ops_sweep.run_table(h['seeds'], h['sigma'], h['learning_rate'], h['weight_decay'], h['action_noise_std'],
                               'cuda')


@pytest.mark.parametrize('R,N', [(1, 2), (3, 5), (4, 64), (2, 2048)])
def test_perturb_sweep_is_the_single_perturb_of_each_runs_seed_and_sigma(R, N):
    from distributedes_b200 import ops, ops_sweep
    rng = np.random.default_rng(R * 10 + N)
    for d0, H, A in ((3, 16, 1), (24, 64, 4), (32, 128, 8)):
        P = orc.param_count(d0, H, A)
        theta = torch.from_numpy((rng.standard_normal((R, P)) * 0.3).astype(np.float32)).cuda()
        h = _hyper(R, rng)
        rows = ops_sweep.nes_perturb_sweep(theta, _table(h), N, 6)
        for r in range(R):
            one = ops.nes_perturb(theta[r].contiguous(), N, h['sigma'][r], h['seeds'][r], 6, member_offset=0)
            assert torch.equal(rows[r * N:(r + 1) * N], one), (d0, H, r)


def _act_case(R, N, d0, A, reps, rng):
    n = R * N
    obs = (rng.standard_normal((n, reps, d0)) * 2).astype(np.float32)
    alive = rng.random((n, reps)) < 0.7
    alive[0] = True
    alive[-1] = False                               # a member with no alive slot
    obs[0, 0, d0 // 2] = np.nan                     # an alive slot's NaN observation gives NaN actions
    stats = np.zeros((R, 2 * d0 + 1), np.float32)
    stats[:, :d0] = rng.normal(0, 0.3, (R, d0))
    stats[:, d0:2 * d0] = rng.uniform(0.5, 1.5, (R, d0))
    stats[:, 2 * d0] = rng.integers(100, 10000, R)
    return (torch.from_numpy(obs).cuda(), torch.from_numpy(alive.astype(np.uint8)).cuda(), torch.from_numpy(stats).cuda())


@pytest.mark.parametrize('H', POLICY_WIDTHS)
@pytest.mark.parametrize('d0,A,reps', [(3, 1, 10), (24, 4, 16), (32, 8, 1), (8, 2, 3)])
@pytest.mark.parametrize('R,N', [(3, 4), (5, 1)])
def test_policy_act_sweep_is_the_single_policy_act_of_each_run(H, d0, A, reps, R, N):
    from distributedes_b200 import ops, ops_sweep
    rng = np.random.default_rng(H * 1000 + d0 * 10 + reps + R)
    P = orc.param_count(d0, H, A)
    rows = torch.from_numpy((rng.standard_normal((R * N, P)) * 0.3).astype(np.float32)).cuda()
    obs, alive, stats = _act_case(R, N, d0, A, reps, rng)
    for use_stats in (False, True):
        for noise in (False, True):
            h = _hyper(R, rng, noise)
            kw = dict(state_dim=d0, hidden=H, action_dim=A, repetitions=reps, clip=1.5, generation=9, t=17)
            part = torch.full((R * N, 2 * d0 + 1), 0.25, dtype=torch.float64, device='cuda')
            act = ops_sweep.policy_act_sweep(rows, obs, alive, _table(h), run_size=N,
                                             obs_stats=stats if use_stats else None, stat_part=part, **kw)
            for r in range(R):
                s = slice(r * N, (r + 1) * N)
                p1 = torch.full((N, 2 * d0 + 1), 0.25, dtype=torch.float64, device='cuda')
                a1 = ops.policy_act(rows[s], obs[s].contiguous(), alive[s].contiguous(), seed=h['seeds'][r],
                                    action_noise_std=h['action_noise_std'][r], member_offset=0,
                                    obs_stats=stats[r] if use_stats else None, stat_part=p1, **kw)
                # bit for bit, NaN included: the bits as integers
                assert torch.equal(act[s].view(torch.int32), a1.view(torch.int32)), (use_stats, noise, r)
                assert torch.equal(part[s].view(torch.int64), p1.view(torch.int64)), (use_stats, noise, r)
            assert torch.isnan(act[0, 0]).all() and not torch.isnan(act[0, 1:]).any()
            assert (act[-1] == 0).all()


@pytest.mark.parametrize('R,N', [(1, 2), (4, 64), (3, 2048)])
def test_parts_reduce_runs_is_the_single_reduce_of_each_run(R, N):
    from distributedes_b200 import ops, ops_sweep
    rng = np.random.default_rng(N + R)
    for d0 in (3, 24, 32):
        parts = torch.from_numpy(rng.standard_normal((R * N, 2 * d0 + 1)) * 100).cuda()
        tot = ops_sweep.obs_parts_reduce_runs(parts, d0, N)
        for r in range(R):
            assert torch.equal(tot[r], ops.obs_parts_reduce(parts[r * N:(r + 1) * N].contiguous(), d0)), (d0, r)


def _walk_batch(seed):
    from distributedes_b200.envs import GymEnvBatch
    return lambda B: GymEnvBatch(sw.SynthWalkEnv, B, seed)


def test_host_sweep_engine_is_r_hostenvengines():
    from distributedes_b200.engine import HostEnvEngine, HostEnvSweepEngine
    H, N, R, reps = 64, 16, 3, 2
    rng = np.random.default_rng(3)
    h = _hyper(R, rng)
    theta0 = np.stack([orc.synthetic_theta(24, H, 4, seed=s) for s in range(R)]).astype(np.float32)
    sweep = HostEnvSweepEngine(env_fn=sw.SynthWalkEnv, batch_env_fn=[_walk_batch(s) for s in h['seeds']], hidden=H,
                               pop_size=N, runs=R, theta0=theta0, repetitions=reps, test_repetitions=3, **h)
    singles = [HostEnvEngine(env_fn=sw.SynthWalkEnv, batch_env_fn=_walk_batch(h['seeds'][r]), hidden=H, pop_size=N,
                             theta0=theta0[r], seed=h['seeds'][r], sigma=h['sigma'][r],
                             learning_rate=h['learning_rate'][r], weight_decay=h['weight_decay'][r],
                             action_noise_std=h['action_noise_std'][r], repetitions=reps, test_repetitions=3)
               for r in range(R)]
    for _ in range(3):
        test = sweep.test_returns()
        sweep.generation()
        for r, e in enumerate(singles):
            assert np.array_equal(test[r], e.test_returns()), r
            e.generation()
            assert sweep.steps_taken[r] == e.steps_taken, r
            for name in ('theta', 'adam_m', 'adam_v', 'fitness_all', 'obs_stats'):
                assert torch.equal(getattr(sweep, name)[r], getattr(e, name)), (name, r)
    assert torch.equal(sweep.state, singles[0].state)


def test_train_sweep_runs_the_host_walk_golden_config_as_train_does():
    from distributedes_b200 import natural_es
    from test_gpu_goldens import synth_walk
    with np.load(os.path.join(os.path.dirname(__file__), 'golden', 'train_host_walk.npz'), allow_pickle=False) as z:
        g = {k: z[k] for k in z.files}
    golden = synth_walk(g)
    configs = []
    for s, sigma in ((int(g['seed']) + 1, 0.05), (None, None), (int(g['seed']) + 7, 0.2)):
        c = copy.copy(golden)
        if s is not None:
            c.seed, c.sigma = s, sigma
        configs.append(c)
    out = natural_es.train_sweep(configs)
    for c, run in zip(configs, out):
        single = natural_es.train(c)
        assert run[0] == single[0] and run[1] == single[1], c.seed
    assert out[1][1] == list(g['train_steps'])
    assert out[1][0] != out[0][0]
