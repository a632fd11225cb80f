"""The CUDA path against the REFERENCE's own outputs (tests/golden/*.npz, written by oracle/make_golden.py from the
reference's verbatim runs) — directly, not through the oracle: Evaluator.eval fitness (utils.py:116-139), and every
train_*.npz, one row each of TRAIN, checked by one of three functions:

* tape: NESEngine generation by generation against natural_es.train() on the synthetic tape (natural_es.py:34-99);
* nes_episodes: natural_es.train() on episodes stepped on the device or on the host, layered on the device's fitness;
* cma_episodes: cma_es.train() on the same episodes, layered on the device's costs, solutions and statistics.

The checks take `device` and `kernels` (default: the current GPU and distributedes_b200.ops), so the table also runs
against tests/cpu_ops on the CPU.

Tolerances of the episode rows: the policy is evaluated in fp32 on the device and in fp64 by the oracle; an episode is
200 steps of a feedback loop, so per-step differences of ~1e-7 grow along the trajectory.  Observed |dR|/|R| <= ~1e-5 on
returns of magnitude ~1e3; the bound used is 2e-4 (ranks may still flip between near-tied members: updates are compared
through the layered protocol, ranks taken from the device's fitness).  The CMA-ES run uses sigma = 1 solutions whose
torque is bang-bang, so later generations amplify rounding: see tests/test_cma_closed_loop_cpu.py."""
import glob
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import host_env_support as hs
from oracle import cma_oracle as cma
from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from oracle import synth_walk as sw

DEV = 'cuda:0'
RTOL = 2e-4


def relnorm(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / np.linalg.norm(b)


@pytest.mark.gpu
@pytest.mark.parametrize('tag', ['pend', 'b64'])
def test_fitness_matches_reference_evaluator(golden_dir, tag):
    """des_nes_eval (fp32 path) == what the reference's Evaluator.eval returned for the same perturbed members: the
    fixture holds -cost of natural_es.py:31-32 for members 0..N-1 of generation 0."""
    from distributedes_b200 import ops
    g = np.load(os.path.join(golden_dir, 'eval_%s.npz' % tag))
    d0, H, A, T = (int(v) for v in g['dims'])
    N, seed, sigma, clip = int(g['N']), int(g['seed']), float(g['sigma']), float(g['clip'])
    obs, target = orc.synthetic_tape(T, d0, A)
    got = ops.nes_eval(torch.from_numpy(g['theta']).to(DEV), torch.from_numpy(obs).to(DEV), torch.from_numpy(target).to(DEV),
                       hidden=H, sigma=sigma, clip=clip, seed=seed, generation=0, member_offset=0, n_local=N,
                       precision='fp32').cpu().numpy().astype(np.float64)
    # the reference runs the forward in fp32 torch on weights perturbed in fp64->fp32; ours regenerates eps with MUFU
    # approximations (|d eps| <= 4e-6): 2e-5 relative on the fitness (measured ~2e-6)
    assert np.max(np.abs(got - g['fitness']) / np.abs(g['fitness'])) < 2e-5
    assert int(g['steps'][0]) == T


# ---- the checks --------------------------------------------------------------------------------------------------------
def tape(g, *, device=None, kernels=None, **opts):
    """NESEngine (opts: normalize_obs, mirrored) against natural_es.train() run verbatim: test rewards
    (natural_es.py:54), gradient after weight decay (:91-93), Adam step and parameters (:94-96), three generations,
    straight from theta0 — populations of 16 / 24 members, where no rank flips.  With the normaliser on, also its
    statistics against the oracle's and the normalised tape the kernels read."""
    from distributedes_b200.engine import NESEngine
    d0, H, A, T = (int(v) for v in g['dims'])
    N, sigma, wd = int(g['N']), float(g['sigma']), float(g['wd'])
    obs, target = orc.synthetic_tape(T, d0, A)
    eng = NESEngine(state_dim=d0, hidden=H, action_dim=A, pop_size=N, theta0=g['theta0'], obs=obs, target=target,
                    sigma=sigma, learning_rate=float(g['lr']), weight_decay=wd, clip=float(g['clip']),
                    seed=int(g['seed']), precision='fp32', device=device, kernels=kernels, **opts)
    stats = orc.ObsStats(d0)
    for gen in range(int(g['gens'])):
        rew = eng.noiseless_fitness()
        assert abs(rew - g['test_rewards'][gen]) < 2e-5 * abs(g['test_rewards'][gen])
        eng.generation()
        grad = eng.partial.cpu().numpy().astype(np.float64) / N / sigma * (1 - wd)
        assert relnorm(grad, g['grad_after_wd'][gen]) <= 2e-5, gen
        if gen >= 1:            # from the second Adam step on the update is well conditioned (the first is ~sign(g))
            assert relnorm(eng.update.cpu().numpy(), g['update'][gen]) <= 2e-5, gen
        assert np.max(np.abs(eng.theta_numpy() - g['theta'][gen])) <= 2e-5
        if opts.get('normalize_obs'):
            stats.merge_tape(obs, N * T)
            sd = eng.stats_state_dict()
            assert np.allclose(sd['m'], stats.m, atol=1e-6) and np.allclose(sd['v'], stats.v, rtol=1e-5)
            assert sd['n'][0] == stats.n
    assert np.array_equal(np.asarray(g['train_steps'][:2]), [0, N * T])
    if opts.get('normalize_obs'):       # the normalised tape the kernels read is (o - m)/sqrt(v + 1e-6)
        ref = np.stack([stats.normalize(o) for o in obs])
        assert np.max(np.abs(eng.k.obs_normalize(eng.obs_raw, eng.obs_stats).cpu().numpy() - ref)) <= 1e-5


def nes_episodes(g, *, config, device=None, kernels=None, **settings):
    """natural_es.train(config(g), with `settings` set on it) against the reference's verbatim train(): the steps
    exactly, test rewards, normaliser statistics, and the parameters, layered: the gradient chain on the device's own
    fitness, then against the golden when no rank flipped."""
    from distributedes_b200 import natural_es
    cfg = config(g)
    for k, v in settings.items():
        setattr(cfg, k, v)
    eng = natural_es.build_engine(cfg, device=device, kernels=kernels)
    assert eng.mirrored == bool(getattr(cfg, 'mirrored', False))
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
    N, seed, sigma = int(g['N']), int(g['seed']), float(g['sigma'])
    theta, opt, P = g['theta0'].copy(), orc.Adam(), g['theta0'].size
    for gen in range(int(g['gens'])):
        assert np.allclose(stats[gen], g['stats'][gen], rtol=5e-4, atol=5e-5)
        s = orc.fitness_shift(fits[gen])
        if eng.mirrored:
            grad = mo.nes_gradient_streamed(s, sigma, seed, gen, P)
        else:
            grad = orc.nes_gradient(orc.noise(seed, gen, 0, N, P), s, sigma)
        theta, _ = orc.nes_update(theta, grad, opt, float(g['wd']), float(g['lr']))
    assert np.max(np.abs(eng.theta_numpy() - theta)) <= 1e-5 * np.max(np.abs(theta - g['theta0']))
    if np.max(np.abs(theta - g['theta'][-1])) <= 2e-6:        # no rank flip happened: equals the reference end to end
        assert np.max(np.abs(eng.theta_numpy() - g['theta'][-1])) <= 1e-5 * np.max(np.abs(g['theta'][-1] - g['theta0']))


def cma_episodes(g, *, config, device=None, kernels=None):
    """cma_es.train(config(g)) against the reference's verbatim cma_es.train().  Every generation is layered: the
    device's costs and statistics are checked against the oracle rolling out the device's own solutions with the
    device's own statistics, and the strategy state against CMAState fed the device's own costs and solutions.  Against
    the golden directly: steps, generation-0 costs and the first two test means (before anything is amplified), ranks
    and m/sigma when no rank flipped, later values within the bounds of the CPU test."""
    from distributedes_b200 import cma_es
    cfg = config(g)
    H, lam, reps, seed, gens = int(g['H']), int(g['lam']), int(g['reps']), int(g['seed']), int(g['gens'])
    worker = cma_es.Worker(0, None, None, None, None, cfg, device=device, kernels=kernels)
    es = cma_es.CMAEvolutionStrategy(cfg.initial_weight, cfg.sigma, lam, seed=seed, device=worker.device, kernels=kernels)
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
    # rollouts: the oracle on the device's own solutions and statistics.  Bang-bang torques make a few members' episodes
    # sensitive to fp32-vs-fp64 rounding once the statistics are on (max 3.8e-3 seen in generation 2 on an H100), while
    # the typical member agrees to ~1e-6: the median is held to 2e-5, the maximum to 2e-2.
    for k, e in enumerate(evals):
        ret, osum, osq, cnt = po.rollouts(e['X'], H, seed, k, np.arange(lam), reps, unpack(e['stats']))
        rel = np.abs(e['cost'] + ret.mean(1)) / np.abs(ret.mean(1))
        assert np.median(rel) < 2e-5 and rel.max() < (RTOL if k == 0 else 2e-2), (k, np.median(rel), rel.max())
        assert e['totals'][6] == cnt and np.allclose(e['totals'][3:6], osq, rtol=RTOL if k == 0 else 2e-2)
    for k, t in enumerate(tests):
        ref_t = po.test_returns(t['sol'], H, seed, k, reps, unpack(t['stats']))
        assert abs(t['ret'].mean() - ref_t.mean()) <= (RTOL if k < 2 else 5e-2) * abs(ref_t.mean()), k
    # merges: Chan merge of the device's totals into the device's previous statistics
    for k, st in enumerate(merged):
        m, v, n = po.merge_totals(unpack(evals[k]['stats']), evals[k]['totals'][:3], evals[k]['totals'][3:6],
                                  evals[k]['totals'][6])
        assert np.allclose(st, np.concatenate([m, v, [n]]), rtol=1e-6, atol=1e-7)
    # strategy state: CMAState fed the device's own solutions and shaped costs
    ref = cma.CMAState(g['theta0'].astype(np.float64), cfg.sigma, lam)
    for k, t in enumerate(tells):
        assert np.array_equal(t['shaped'], orc.fitness_shift(evals[k]['cost']).astype(np.float32))
        ref.tell(evals[k]['X'].astype(np.float64), t['shaped'])
        assert np.linalg.norm(t['m'] - ref.m) <= 2e-5 * np.linalg.norm(ref.m)
        assert np.linalg.norm(t['pc'] - ref.pc) <= 2e-5 * np.linalg.norm(ref.pc)
        assert abs(t['sigma'] - ref.sigma) <= 2e-5 * ref.sigma
    # against the golden itself
    z_err = 4e-6 * (1 + np.abs(g['solutions'][0] - g['theta0'][None, :]))
    assert np.all(np.abs(evals[0]['X'] - g['solutions'][0]) <= z_err * float(g['sigma']) + 1e-6)
    assert np.allclose(-evals[0]['cost'], -g['costs'][0], rtol=1e-3)
    assert np.allclose(rewards[:2], g['test_rewards'][:2], rtol=RTOL)
    # test() call k + 1 runs the best member of generation k: comparable with the golden when both chose the same member
    # (the golden pins the argmin of the generations it told)
    for k in range(gens):
        if int(np.argmin(evals[k]['cost'])) == int(np.argmin(g['costs'][k])):
            assert abs(rewards[k + 1] - g['test_rewards'][k + 1]) <= 5e-2 * abs(g['test_rewards'][k + 1]), k
    assert np.allclose(merged[-1], g['stats'][-1], rtol=1e-2, atol=2e-5)
    if all(np.array_equal(t['shaped'], g['shaped'][k].astype(np.float32)) for k, t in enumerate(tells)):
        assert np.linalg.norm(tells[-1]['m'] - g['m'][-1]) <= 2e-5 * np.linalg.norm(g['m'][-1])
        assert abs(tells[-1]['sigma'] - float(g['sigmas'][-1])) <= 2e-5 * float(g['sigmas'][-1])


# ---- the configs of the episode rows -----------------------------------------------------------------------------------
def _golden_run(cfg, g):
    """The fixture's theta0, population, sigma, seed, repetitions and (NES) learning rate."""
    cfg.initial_weight = g['theta0'].copy()
    cfg.pop_size = int(g['N'] if 'N' in g else g['lam'])
    cfg.sigma, cfg.seed = float(g['sigma']), int(g['seed'])
    if 'lr' in g:
        cfg.learning_rate = float(g['lr'])
    cfg.repetitions = cfg.test_repetitions = int(g['reps'])
    return cfg


def _pendulum_run(cfg, g):
    """Pendulum episodes all last 200 steps: the collection after the fixture's last update (NES) or tell (CMA-ES) is
    the first to pass max_steps."""
    _golden_run(cfg, g)
    cfg.max_steps = (int(g['gens']) + 1) * cfg.pop_size * cfg.repetitions * 200 - 1
    return cfg


def device_rollouts(g):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    return _pendulum_run(ClosedLoopPendulumConfig(int(g['H'])), g)


def host_pendulum(g):
    from distributedes_b200.config import HostEnvConfig
    seed = int(g['seed'])
    return _pendulum_run(HostEnvConfig(hs.PendulumProbe, hidden_size=int(g['H']), clip=2.0, task='Pendulum-v0',
                                       batch_env_fn=lambda B: po.PendulumBatch(B, seed)), g)


def synth_walk(g):
    """SynthWalk-v0 through envs.GymEnvBatch: episodes of varying length."""
    from distributedes_b200.config import HostEnvConfig
    cfg = _golden_run(HostEnvConfig(sw.SynthWalkEnv, hidden_size=int(g['H']), clip=1.0, task='SynthWalk-v0'), g)
    cfg.max_steps = int(g['train_steps'][-1])            # the collection after the last update ends the run
    return cfg


TRAIN = [
    pytest.param('train_pend', tape, {}, id='pend'),
    pytest.param('train_b64', tape, {}, id='b64'),
    pytest.param('train_norm_pend', tape, dict(normalize_obs=True), id='norm_pend'),
    pytest.param('train_norm_b64', tape, dict(normalize_obs=True), id='norm_b64'),
    pytest.param('train_b64_mirrored', tape, dict(mirrored=True), id='b64_mirrored'),
    pytest.param('train_closed_pend', nes_episodes, dict(config=device_rollouts), id='closed_pend'),
    pytest.param('train_closed_pend', nes_episodes, dict(config=host_pendulum), id='closed_pend_host'),
    pytest.param('train_closed_mirrored_pend', nes_episodes, dict(config=device_rollouts, mirrored=True),
                 id='closed_mirrored_pend'),
    pytest.param('train_host_walk', nes_episodes, dict(config=synth_walk), id='host_walk'),
    pytest.param('train_cma_closed_pend', cma_episodes, dict(config=device_rollouts), id='cma_closed_pend'),
    pytest.param('train_cma_closed_pend', cma_episodes, dict(config=host_pendulum), id='cma_closed_pend_host'),
]


@pytest.mark.gpu
@pytest.mark.parametrize('fixture,check,opts', TRAIN)
def test_generations_match_reference_train(golden_dir, fixture, check, opts):
    check(np.load(os.path.join(golden_dir, fixture + '.npz')), **opts)


def test_every_training_golden_has_a_row(golden_dir):
    on_disk = {os.path.basename(p)[:-len('.npz')] for p in glob.glob(os.path.join(golden_dir, 'train_*.npz'))}
    assert on_disk == {row.values[0] for row in TRAIN}


@pytest.mark.gpu
def test_host_normaliser_surface_feeds_the_device_path():
    """utils.StaticNormalizer / SharedStats with NON-empty statistics: Evaluator.eval normalises the tape on the device
    with the offline statistics (utils.py:48-51,131) and accumulates the online ones (utils.py:68-73)."""
    from distributedes_b200.config import BipedalWalkerConfig
    from distributedes_b200.utils import Evaluator, SharedStats, StaticNormalizer
    cfg = BipedalWalkerConfig(hidden_size=64, tape_len=64)
    env = cfg.env_fn()
    norm = StaticNormalizer(cfg.state_dim)
    warm = SharedStats(cfg.state_dim)
    for o in env.obs[:40]:
        warm.feed(o)
    norm.offline_stats.load(warm)
    ev = Evaluator(cfg, norm)
    cost, steps = ev.eval(cfg.initial_weight)
    stats = orc.ObsStats(cfg.state_dim)
    stats.m, stats.v, stats.n = warm.m.copy(), warm.v.copy(), np.float32(warm.n[0])
    nobs = np.stack([stats.normalize(o) for o in env.obs]).astype(np.float32)
    ref = orc.tape_fitness(orc.forward(cfg.initial_weight, nobs, 24, 64, 4), env.target, 1.0)
    assert steps == 64 and abs(-cost - ref) < 5e-5 * abs(ref)
    assert norm.online_stats.n[0] == 64 * cfg.repetitions
    assert np.allclose(norm.online_stats.m, env.obs.mean(0), atol=1e-5)
