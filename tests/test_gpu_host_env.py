"""des_policy_act (the population's policy step for environments stepped on the host) and the training surfaces over it:
the fp64 forward, the action-noise stream, dead slots, the statistics order, shard invariance, host-stepped Pendulum-v0
against the oracle and the goldens of the device rollout (train_closed_pend.npz, train_cma_closed_pend.npz), and
natural_es.train on SynthWalk-v0 against the reference's verbatim run (train_host_walk.npz).

Tolerance of the actions: the fp32 forward differs from the fp64 one by fp32 rounding of the FMA chains plus the MUFU
tanh's ~2e-7 absolute error per unit; |W3| sums to O(1) for these weights, so |da| stays below ~1e-5 (3e-5 (1 + |a|) is
used).  Action noise adds the MUFU Box-Muller error, <= 4e-6 (1 + |z|) times the std."""
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from oracle import synth_walk as sw

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import host_env_support as hs        # noqa: E402

RTOL = 2e-4


def dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).cuda()


def _rows(d0, H, A, n, seed):
    theta = orc.synthetic_theta(d0, H, A, seed=seed)
    return orc.perturb(theta, 0.1, orc.noise(seed, 0, 0, n, theta.size))


def _stats(d0, rs):
    return (rs.randn(d0).astype(np.float32) * 0.3, (rs.rand(d0) + 0.5).astype(np.float32), np.float32(1000))


@pytest.mark.parametrize('H', [16, 32, 64, 96, 128])
@pytest.mark.parametrize('d0,A', [(3, 1), (8, 2), (24, 4), (32, 8)])
@pytest.mark.parametrize('reps', [1, 10, 16])
def test_policy_act_matches_fp64_forward(H, d0, A, reps):
    from distributedes_b200 import ops
    n, seed, gen, off = 7, 3 + H, 2, 5
    rs = np.random.RandomState(H * 100 + d0 * 10 + reps)
    rows = _rows(d0, H, A, n, seed)
    obs = (rs.randn(n, reps, d0) * 2).astype(np.float32)
    alive = rs.rand(n, reps) < 0.7
    alive[0] = True
    stats = _stats(d0, rs)
    for use_stats in (False, True):
        for noise in (0.0, 0.3):
            st = dev(np.concatenate([stats[0], stats[1], [stats[2]]])) if use_stats else None
            part = torch.zeros((n, 2 * d0 + 1), dtype=torch.float64, device='cuda')
            act = ops.policy_act(dev(rows), dev(obs), dev(alive, torch.uint8), state_dim=d0, hidden=H, action_dim=A,
                                 repetitions=reps, clip=1.5, action_noise_std=noise, seed=seed, generation=gen,
                                 member_offset=off, t=4, obs_stats=st, stat_part=part).cpu().numpy()
            ref = hs.policy_actions(rows, obs, alive, d0, H, A, 1.5, stats if use_stats else None, noise, seed, gen, off,
                                    4)
            assert act.shape == (n, reps, A)
            assert np.all(act[~alive] == 0.0)
            assert np.max(np.abs(act - ref) / (1 + np.abs(ref))) < 3e-5, (use_stats, noise)
            want = np.zeros((n, 2 * d0 + 1))
            hs.accumulate_stats(want, obs, alive)
            assert np.array_equal(part.cpu().numpy(), want)


def test_action_noise_is_the_counter_stream_and_statistics_accumulate_in_step_order():
    """Zero weights: the action is clip(std * z), z the documented counter normals (quads beyond the fourth action
    included); two launches accumulate the statistics in (step, repetition) order, bit for bit."""
    from distributedes_b200 import ops
    d0, H, A, reps, n = 5, 32, 8, 16, 3
    P = orc.param_count(d0, H, A)
    rows = dev(np.zeros((n, P)))
    rs = np.random.RandomState(1)
    part = torch.zeros((n, 2 * d0 + 1), dtype=torch.float64, device='cuda')
    want = np.zeros((n, 2 * d0 + 1))
    for t in (0, 7):
        obs = rs.randn(n, reps, d0).astype(np.float32)
        alive = rs.rand(n, reps) < 0.8
        act = ops.policy_act(rows, dev(obs), dev(alive, torch.uint8), state_dim=d0, hidden=H, action_dim=A,
                             repetitions=reps, clip=10.0, action_noise_std=1.0, seed=99, generation=6, member_offset=11,
                             t=t, stat_part=part).cpu().numpy()
        z = hs.action_noise(99, 6, np.arange(11, 11 + n), reps, t, A)
        assert np.all(np.abs(act - z)[alive] <= 4e-6 * (1 + np.abs(z[alive])))
        assert np.all(act[~alive] == 0)
        hs.accumulate_stats(want, obs, alive)
        assert np.array_equal(part.cpu().numpy(), want)
    tot = ops.obs_parts_reduce(part, d0).cpu().numpy()
    assert np.array_equal(tot, want[0] + want[1] + want[2])


def test_policy_act_is_shard_invariant():
    from distributedes_b200 import ops
    d0, H, A, reps, n = 24, 64, 4, 10, 9
    rows = dev(_rows(d0, H, A, n, 4))
    rs = np.random.RandomState(2)
    obs, alive = dev(rs.randn(n, reps, d0)), dev(rs.rand(n, reps) < 0.6, torch.uint8)
    st = dev(np.concatenate(list(_stats(d0, rs)[:2]) + [[50.0]]))
    kw = dict(state_dim=d0, hidden=H, action_dim=A, repetitions=reps, clip=1.0, action_noise_std=0.1, seed=3,
              generation=1, t=12, obs_stats=st)
    parts = [torch.zeros((k, 2 * d0 + 1), dtype=torch.float64, device='cuda') for k in (n, 4, n - 4)]
    whole = ops.policy_act(rows, obs, alive, member_offset=0, stat_part=parts[0], **kw)
    a = ops.policy_act(rows[:4].contiguous(), obs[:4].contiguous(), alive[:4].contiguous(), member_offset=0,
                       stat_part=parts[1], **kw)
    b = ops.policy_act(rows[4:].contiguous(), obs[4:].contiguous(), alive[4:].contiguous(), member_offset=4,
                       stat_part=parts[2], **kw)
    assert torch.equal(whole, torch.cat([a, b])) and torch.equal(parts[0], torch.cat(parts[1:]))


def test_policy_act_rejects_bad_arguments():
    from distributedes_b200 import ops
    rows = dev(np.zeros((2, orc.param_count(24, 64, 4))))
    obs, alive = dev(np.zeros((2, 17, 24))), dev(np.ones((2, 17)), torch.uint8)
    with pytest.raises(RuntimeError, match='repetitions must be in'):
        ops.policy_act(rows, obs, alive, state_dim=24, hidden=64, action_dim=4, repetitions=17, clip=1.0, seed=0,
                       generation=0, t=0)
    with pytest.raises(RuntimeError, match='MLP needs'):
        ops.policy_act(rows, obs[:, :2].contiguous(), alive[:, :2].contiguous(), state_dim=24, hidden=32, action_dim=4,
                       repetitions=2, clip=1.0, seed=0, generation=0, t=0)


# ---- host-stepped Pendulum-v0 against the device rollout's oracle and goldens ------------------------------------------
class PendulumProbe:
    """Pendulum-v0's spaces, for the configs' probe; the episodes run in host_env_support.PendulumBatch."""
    class _Box:
        def __init__(self, n):
            self.shape = (n,)
    observation_space, action_space = _Box(3), _Box(1)


def _pendulum_engine(H, N, reps, seed, theta0, **kw):
    from distributedes_b200.engine import HostEnvEngine
    return HostEnvEngine(env_fn=PendulumProbe, batch_env_fn=lambda B: hs.PendulumBatch(B, seed), hidden=H, pop_size=N,
                         theta0=theta0, sigma=0.1, learning_rate=0.1, repetitions=reps, clip=2.0, seed=seed, **kw)


def test_host_stepped_pendulum_matches_the_rollout_oracle():
    H, N, reps, seed = 64, 12, 10, 4
    theta = orc.synthetic_theta(3, H, 1, seed=2)
    eng = _pendulum_engine(H, N, reps, seed, theta)
    stats = (np.array([-0.2, 0.01, 0.3], np.float32), np.array([0.5, 0.4, 20.0], np.float32), np.float32(32000))
    eng.obs_stats.copy_(dev(np.concatenate([stats[0], stats[1], [stats[2]]])))
    eng.generation_index = 1
    fit = eng.evaluate().cpu().numpy().astype(np.float64)
    ref, (osum, osq, cnt) = po.closed_fitness(theta, H, 0.1, seed, 1, 0, N, reps, stats)
    assert np.max(np.abs(fit - ref) / np.abs(ref)) < RTOL
    assert eng.steps_taken == N * reps * 200
    t = eng.obs_totals.cpu().numpy()
    assert t[6] == cnt and np.allclose(t[:3], osum, rtol=RTOL, atol=1e-3 * cnt ** 0.5) and np.allclose(t[3:6], osq,
                                                                                                      rtol=RTOL)
    ref_t = po.test_returns(theta, H, seed, 1, reps, stats)
    assert np.max(np.abs(eng.test_returns() - ref_t) / np.abs(ref_t)) < RTOL


def test_two_shards_on_one_gpu_equal_one_shard():
    """Episodes keyed by the global member: two shards' fitness and statistics rows equal the whole population's."""
    from distributedes_b200 import ops
    from distributedes_b200.engine import HostEpisodes
    H, N, reps, seed, gen = 32, 11, 10, 6, 3
    rows = ops.nes_perturb(dev(orc.synthetic_theta(3, H, 1, seed=1)), N, 0.1, seed, gen)
    out = []
    for lo, hi in ((0, N), (0, 5), (5, N)):
        part = torch.zeros((hi - lo, 7), dtype=torch.float64, device='cuda')
        ep = HostEpisodes(ops, 'cuda', hs.PendulumBatch((hi - lo) * reps, seed, horizon=60), hi - lo, reps, 3, H, 1, 2.0,
                          0.2, seed)
        ret, steps = ep.run(rows[lo:hi].contiguous(), generation=gen, member_offset=lo, stat_part=part)
        out.append((ret.mean(1).astype(np.float32), part.cpu().numpy(), steps))
    assert np.array_equal(out[0][0], np.concatenate([out[1][0], out[2][0]]))
    assert np.array_equal(out[0][1], np.concatenate([out[1][1], out[2][1]]))
    assert out[0][2] == out[1][2] + out[2][2] == N * reps * 60


def test_natural_es_train_over_host_stepped_pendulum_matches_reference_golden():
    """The assertions of test_train_on_closed_loop_pendulum_matches_reference_golden, with Pendulum-v0 stepped on the
    host (natural_es.train(HostEnvConfig(...)))."""
    from distributedes_b200 import natural_es
    from distributedes_b200.config import HostEnvConfig
    g = np.load(os.path.join(HERE, 'golden', 'train_closed_pend.npz'))
    H, N, reps, seed, gens = int(g['H']), int(g['N']), int(g['reps']), int(g['seed']), int(g['gens'])
    cfg = HostEnvConfig(PendulumProbe, hidden_size=H, clip=2.0, task='Pendulum-v0',
                        batch_env_fn=lambda B: hs.PendulumBatch(B, seed))
    cfg.initial_weight = g['theta0'].copy()
    cfg.pop_size, cfg.sigma, cfg.learning_rate, cfg.seed = N, float(g['sigma']), float(g['lr']), seed
    cfg.repetitions = cfg.test_repetitions = reps
    cfg.max_steps = (gens + 1) * N * reps * 200 - 1
    eng = natural_es.build_engine(cfg)
    fits, stats = [], []
    real_rank, real_apply = eng.rank_and_reduce, eng.apply

    def spy_rank():
        fits.append(eng.fitness_all.cpu().numpy().astype(np.float64))
        return real_rank()

    def spy_apply():
        real_apply()
        stats.append(eng.obs_stats.cpu().numpy().copy())
    eng.rank_and_reduce, eng.apply = spy_rank, spy_apply
    rewards, steps, _ = natural_es.train(cfg, engine=eng)
    assert steps == list(g['train_steps'])
    assert np.allclose(rewards, g['test_rewards'], rtol=RTOL)
    theta, opt, P = g['theta0'].copy(), orc.Adam(), g['theta0'].size
    for gen in range(gens):
        assert np.allclose(stats[gen], g['stats'][gen], rtol=5e-4, atol=5e-5)
        s = orc.fitness_shift(fits[gen])
        grad = orc.nes_gradient(orc.noise(seed, gen, 0, N, P), s, float(g['sigma']))
        theta, _ = orc.nes_update(theta, grad, opt, float(g['wd']), float(g['lr']))
    assert np.max(np.abs(eng.theta_numpy() - theta)) <= 1e-5 * np.max(np.abs(theta - g['theta0']))
    if np.max(np.abs(theta - g['theta'][-1])) <= 2e-6:
        assert np.max(np.abs(eng.theta_numpy() - g['theta'][-1])) <= 1e-5 * np.max(np.abs(g['theta'][-1] - g['theta0']))


def test_cma_train_over_host_stepped_pendulum_matches_reference_golden():
    """The assertions of test_cma_train_on_closed_loop_pendulum_matches_reference_golden at H = 16, with Pendulum-v0
    stepped on the host (cma_es.train(HostEnvConfig(...)))."""
    from oracle import cma_oracle as cma
    from distributedes_b200 import cma_es
    from distributedes_b200.config import HostEnvConfig
    g = np.load(os.path.join(HERE, 'golden', 'train_cma_closed_pend.npz'))
    H, lam, reps, seed, gens = int(g['H']), int(g['lam']), int(g['reps']), int(g['seed']), int(g['gens'])
    cfg = HostEnvConfig(PendulumProbe, hidden_size=H, clip=2.0, task='Pendulum-v0',
                        batch_env_fn=lambda B: hs.PendulumBatch(B, seed))
    cfg.initial_weight = g['theta0'].copy()
    cfg.pop_size, cfg.sigma, cfg.seed = lam, float(g['sigma']), seed
    cfg.max_steps = (gens + 1) * lam * reps * 200 - 1
    worker = cma_es.Worker(0, None, None, None, None, cfg)
    es = cma_es.CMAEvolutionStrategy(cfg.initial_weight, cfg.sigma, lam, seed=seed, device=worker.device)
    evals, tells, tests, merged = [], [], [], []
    real_run, real_tell, real_test, real_merge = worker.run, es.tell, worker.test_returns, worker.merge_obs_stats

    def spy_run(solutions, member_offset=0, generation=0):
        st = worker.obs_stats.cpu().numpy().copy()
        cost = real_run(solutions, member_offset, generation)
        evals.append(dict(X=solutions.cpu().numpy().copy(), stats=st, cost=cost.cpu().numpy().astype(np.float64),
                          totals=worker.obs_totals.cpu().numpy().copy()))
        return cost

    def spy_tell(solutions, cost):
        out = real_tell(solutions, cost)
        tells.append(dict(shaped=cost.cpu().numpy().astype(np.float64), m=es.m.cpu().numpy(), sigma=es.sigma,
                          pc=es.pc.cpu().numpy()))
        return out

    def spy_test(solution, repetitions):
        st = worker.obs_stats.cpu().numpy().copy()
        ret = real_test(solution, repetitions)
        tests.append(dict(sol=solution.reshape(-1).cpu().numpy().copy(), stats=st, ret=ret))
        return ret

    def spy_merge(es_):
        real_merge(es_)
        merged.append(worker.obs_stats.cpu().numpy().copy())
    worker.run, es.tell, worker.test_returns, worker.merge_obs_stats = spy_run, spy_tell, spy_test, spy_merge
    rewards, steps, _ = cma_es.train(cfg, worker=worker, es=es)
    assert steps == list(g['train_steps']) and len(evals) == gens + 1 and len(tells) == len(merged) == gens

    def unpack(a):
        return (a[:3], a[3:6], a[6])
    for k, e in enumerate(evals):
        ret, osum, osq, cnt = po.rollouts(e['X'], H, seed, k, np.arange(lam), reps, unpack(e['stats']))
        rel = np.abs(e['cost'] + ret.mean(1)) / np.abs(ret.mean(1))
        assert np.median(rel) < 2e-5 and rel.max() < (RTOL if k == 0 else 2e-2), (k, np.median(rel), rel.max())
        assert e['totals'][6] == cnt and np.allclose(e['totals'][3:6], osq, rtol=RTOL if k == 0 else 2e-2)
    for k, t in enumerate(tests):
        ref_t = po.test_returns(t['sol'], H, seed, k, reps, unpack(t['stats']))
        assert abs(t['ret'].mean() - ref_t.mean()) <= (RTOL if k < 2 else 5e-2) * abs(ref_t.mean()), k
    for k, st in enumerate(merged):
        m, v, n = po.merge_totals(unpack(evals[k]['stats']), evals[k]['totals'][:3], evals[k]['totals'][3:6],
                                  evals[k]['totals'][6])
        assert np.allclose(st, np.concatenate([m, v, [n]]), rtol=1e-6, atol=1e-7)
    ref = cma.CMAState(g['theta0'].astype(np.float64), cfg.sigma, lam)
    for k, t in enumerate(tells):
        assert np.array_equal(t['shaped'], orc.fitness_shift(evals[k]['cost']).astype(np.float32))
        ref.tell(evals[k]['X'].astype(np.float64), t['shaped'])
        assert np.linalg.norm(t['m'] - ref.m) <= 2e-5 * np.linalg.norm(ref.m)
        assert np.linalg.norm(t['pc'] - ref.pc) <= 2e-5 * np.linalg.norm(ref.pc)
        assert abs(t['sigma'] - ref.sigma) <= 2e-5 * ref.sigma
    z_err = 4e-6 * (1 + np.abs(g['solutions'][0] - g['theta0'][None, :]))
    assert np.all(np.abs(evals[0]['X'] - g['solutions'][0]) <= z_err * float(g['sigma']) + 1e-6)
    assert np.allclose(-evals[0]['cost'], -g['costs'][0], rtol=1e-3)
    assert np.allclose(rewards[:2], g['test_rewards'][:2], rtol=RTOL)
    for k in range(gens):
        if int(np.argmin(evals[k]['cost'])) == int(np.argmin(g['costs'][k])):
            assert abs(rewards[k + 1] - g['test_rewards'][k + 1]) <= 5e-2 * abs(g['test_rewards'][k + 1]), k
    assert np.allclose(merged[-1], g['stats'][-1], rtol=1e-2, atol=2e-5)
    if all(np.array_equal(t['shaped'], g['shaped'][k].astype(np.float32)) for k, t in enumerate(tells)):
        assert np.linalg.norm(tells[-1]['m'] - g['m'][-1]) <= 2e-5 * np.linalg.norm(g['m'][-1])
        assert abs(tells[-1]['sigma'] - float(g['sigmas'][-1])) <= 2e-5 * float(g['sigmas'][-1])


def test_natural_es_train_on_synth_walk_matches_reference_golden():
    """natural_es.train(HostEnvConfig(SynthWalkEnv)) through envs.GymEnvBatch against the reference's verbatim train():
    the real step counts exactly, the test rewards, the statistics and the parameters layered on the device's own
    fitness."""
    from distributedes_b200 import natural_es
    from distributedes_b200.config import HostEnvConfig
    g = np.load(os.path.join(HERE, 'golden', 'train_host_walk.npz'))
    H, N, reps, seed, gens = int(g['H']), int(g['N']), int(g['reps']), int(g['seed']), int(g['gens'])
    cfg = HostEnvConfig(sw.SynthWalkEnv, hidden_size=H, clip=1.0, task='SynthWalk-v0')
    cfg.initial_weight = g['theta0'].copy()
    cfg.pop_size, cfg.sigma, cfg.learning_rate, cfg.seed = N, float(g['sigma']), float(g['lr']), seed
    cfg.max_steps = int(g['train_steps'][-1])            # the collection after the last update ends the run
    eng = natural_es.build_engine(cfg)
    fits, stats = [], []
    real_rank, real_apply = eng.rank_and_reduce, eng.apply

    def spy_rank():
        fits.append(eng.fitness_all.cpu().numpy().astype(np.float64))
        return real_rank()

    def spy_apply():
        real_apply()
        stats.append(eng.obs_stats.cpu().numpy().copy())
    eng.rank_and_reduce, eng.apply = spy_rank, spy_apply
    rewards, steps, _ = natural_es.train(cfg, engine=eng)
    assert steps == list(g['train_steps'])
    assert np.allclose(rewards, g['test_rewards'], rtol=RTOL)
    theta, opt, P = g['theta0'].copy(), orc.Adam(), g['theta0'].size
    for gen in range(gens):
        assert np.allclose(stats[gen], g['stats'][gen], rtol=5e-4, atol=5e-5)
        grad = orc.nes_gradient(orc.noise(seed, gen, 0, N, P), orc.fitness_shift(fits[gen]), float(g['sigma']))
        theta, _ = orc.nes_update(theta, grad, opt, float(g['wd']), float(g['lr']))
    assert np.max(np.abs(eng.theta_numpy() - theta)) <= 1e-5 * np.max(np.abs(theta - g['theta0']))
    if np.max(np.abs(theta - g['theta'][-1])) <= 2e-6:
        assert np.max(np.abs(eng.theta_numpy() - g['theta'][-1])) <= 1e-5 * np.max(np.abs(g['theta'][-1] - g['theta0']))


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpu_host_env_equals_one_gpu(tmp_path):
    import subprocess
    script = os.path.join(HERE, 'mp_host_env_worker.py')
    out = str(tmp_path)
    subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
                    '127.0.0.1', '--master-port', '29767', script, out], check=True, timeout=600)
    r0, r1 = np.load(os.path.join(out, 'rank0.npz')), np.load(os.path.join(out, 'rank1.npz'))
    for k in ('fit', 'steps', 'stats', 'theta'):
        assert np.array_equal(r0[k], r1[k]), k
    import importlib.util
    spec = importlib.util.spec_from_file_location('mp_host_env_worker', script)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    one = mod.run()
    assert np.array_equal(one['fit'], r0['fit']) and np.array_equal(one['steps'], r0['steps'])
    assert np.allclose(one['stats'], r0['stats'], rtol=1e-6, atol=1e-7)
