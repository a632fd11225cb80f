"""Closed-loop rollouts (SURVEY 8f row 3) on CPU: the oracle against the reference's own natural_es.train() run
verbatim on its PendulumConfig (tests/golden/train_closed_pend.npz, oracle/make_golden.py::train_env), and
the world_size-2 host logic of engine.RolloutEngine under gloo."""
import os

import numpy as np

import cpu_ops
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from ranks import spawn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(REPO, 'tests', 'golden', 'train_closed_pend.npz')


def oracle_chain(theta, H, N, reps, seed, sigma, lr, wd, gens, horizon=po.HORIZON):
    """Single-process chain of closed-loop generations with the oracle; yields per-generation records."""
    P = theta.size
    stats = (np.zeros(3, np.float32), np.zeros(3, np.float32), np.float32(0))
    opt = orc.Adam()
    for gen in range(gens):
        test = po.test_returns(theta, H, seed, gen, reps, stats, horizon)
        fit, (osum, osq, cnt) = po.closed_fitness(theta, H, sigma, seed, gen, 0, N, reps, stats, horizon)
        stats = po.merge_totals(stats, osum, osq, cnt)
        grad = orc.nes_gradient(orc.noise(seed, gen, 0, N, P), orc.fitness_shift(fit), sigma)
        theta, upd = orc.nes_update(theta, grad, opt, wd, lr)
        yield dict(test=test, fitness=fit, stats=np.concatenate([stats[0], stats[1], [stats[2]]]),
                   grad_after_wd=grad - wd * grad, theta=theta)


def test_oracle_matches_verbatim_reference_train_on_pendulum():
    g = np.load(GOLD)
    H, N, reps, seed, gens = int(g['H']), int(g['N']), int(g['reps']), int(g['seed']), int(g['gens'])
    assert (H, N, reps) == (64, 16, 10)                       # BASELINE configs[0]
    recs = list(oracle_chain(g['theta0'].copy(), H, N, reps, seed, float(g['sigma']), float(g['lr']), float(g['wd']), gens))
    assert list(g['train_steps']) == [k * N * reps * po.HORIZON for k in range(gens + 1)]
    for gen, r in enumerate(recs):
        # test(): mean return of the 10 noiseless episodes (natural_es.py:54, 101-110)
        assert abs(r['test'].mean() - g['test_rewards'][gen]) <= 1e-5 * abs(g['test_rewards'][gen])
        # normaliser statistics after the merge (natural_es.py:85-89); the reference accumulates them in fp32
        assert np.allclose(r['stats'], g['stats'][gen], rtol=2e-4, atol=2e-5)
        # gradient: identical ranks -> agreement to fp64 rounding in generation 0, fp32-normaliser noise afterwards
        scale = np.abs(g['grad_after_wd'][gen]).max()
        assert np.abs(r['grad_after_wd'] - g['grad_after_wd'][gen]).max() <= (1e-12 if gen == 0 else 1e-5) * scale
        assert np.abs(r['theta'] - g['theta'][gen]).max() <= 2e-6


def test_reset_states_are_in_range_and_distinct():
    th, thd = po.reset_states(3, 1, np.arange(64), 10)
    assert th.shape == (64, 10) and np.all(np.abs(th) < np.pi) and np.all(np.abs(thd) < 1)
    assert len(np.unique(th)) == th.size
    th2, _ = po.reset_states(3, 2, np.arange(64), 10)
    assert not np.any(th == th2)


def _worker(N, gens):
    from distributedes_b200.engine import RolloutEngine
    theta0 = orc.synthetic_theta(3, 32, 1)
    eng = RolloutEngine(hidden=32, pop_size=N, theta0=theta0, sigma=0.1, learning_rate=0.1, repetitions=2, horizon=20,
                        seed=13, device='cpu', kernels=cpu_ops)
    tests = []
    for _ in range(gens):
        tests.append(eng.test_returns())
        eng.generation()
    return dict(theta=eng.theta.numpy(), stats=eng.obs_stats.numpy(), fit=eng.fitness_all.numpy(), tests=np.stack(tests))


def test_rollout_engine_sharded_equals_single_process():
    """Ragged 2-rank split: fitness all-gather, fp64 observation-total all-reduce, identical update on both ranks."""
    N, world, gens = 7, 2, 2
    res = spawn(world, _worker, N, gens)
    for k in ('theta', 'stats', 'fit', 'tests'):
        assert np.array_equal(res[0][k], res[1][k]), k
    recs = list(oracle_chain(orc.synthetic_theta(3, 32, 1), 32, N, 2, 13, 0.1, 0.1, 0.005, gens, horizon=20))
    assert np.allclose(res[0]['fit'], recs[-1]['fitness'], rtol=1e-6)
    assert np.allclose(res[0]['stats'], recs[-1]['stats'], rtol=1e-5, atol=1e-6)
    assert np.allclose(res[0]['tests'][1], recs[1]['test'], rtol=1e-6)
    assert np.max(np.abs(res[0]['theta'] - recs[-1]['theta'])) <= 2e-6


def _train_worker():
    """natural_es.train() — the reference-facing loop — on two ranks under gloo, closed loop, oracle-backed kernels."""
    from distributedes_b200 import natural_es
    from distributedes_b200.config import ClosedLoopPendulumConfig
    g = np.load(GOLD)
    cfg = ClosedLoopPendulumConfig(hidden_size=int(g['H']))
    cfg.initial_weight = g['theta0'].copy()
    cfg.pop_size, cfg.sigma, cfg.learning_rate, cfg.seed = int(g['N']), float(g['sigma']), float(g['lr']), int(g['seed'])
    cfg.max_steps = (int(g['gens']) + 1) * cfg.pop_size * cfg.repetitions * 200 - 1
    eng = natural_es.build_engine(cfg, device='cpu', kernels=cpu_ops)
    rewards, steps, stamps = natural_es.train(cfg, engine=eng)
    return dict(rewards=np.asarray(rewards), steps=np.asarray(steps), theta=eng.theta.numpy(), n_stamps=len(stamps))


def test_train_surface_on_two_ranks_reproduces_the_reference_golden():
    """BASELINE configs[0] through natural_es.train(ClosedLoopPendulumConfig) on 2 ranks (8 members each): the returned
    [rewards, steps, timestamps] triple and the final parameters equal the reference's verbatim run."""
    g = np.load(GOLD)
    r = spawn(2, _train_worker)
    for k in ('rewards', 'steps', 'theta'):
        assert np.array_equal(r[0][k], r[1][k]), k
    assert list(r[0]['steps']) == list(g['train_steps']) and int(r[0]['n_stamps']) == len(g['train_steps'])
    assert np.allclose(r[0]['rewards'], g['test_rewards'], rtol=1e-5)
    assert np.max(np.abs(r[0]['theta'] - g['theta'][-1])) <= 2e-6
