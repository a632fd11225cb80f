"""Closed-loop CMA-ES on CPU: the oracle chain against the reference's own cma_es.train() run verbatim on its
PendulumConfig(hidden_size=16) (tests/golden/train_cma_closed_pend.npz, oracle/make_golden.py::train_cma), the
sharded host logic of cma_es.train under gloo, and the C ABI's argument checks for des_rollout_eval_solutions."""
import os

import numpy as np
import pytest
import torch.distributed as dist

import cpu_ops
from lib_fixture import lib  # noqa: F401
from oracle import cma_oracle as cma
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from ranks import spawn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(REPO, 'tests', 'golden', 'train_cma_closed_pend.npz')


def oracle_cma_chain(theta0, H, lam, reps, seed, sigma, gens, horizon=po.HORIZON, stats_feed=None):
    """cma_es.py:31-100 with the oracles: CMAState for pycma, explicit-row rollouts for the workers, Chan merges of the raw
    observation sums for SharedStats.  Returns per-tell records and the test returns of every test() call.

    stats_feed (layered check): after the k-th merge, continue from stats_feed[k] instead of the chain's own result."""
    st = cma.CMAState(np.asarray(theta0, np.float64), sigma, lam)
    stats = (np.zeros(3, np.float32), np.zeros(3, np.float32), np.float32(0))
    tests = [po.test_returns(theta0, H, seed, 0, reps, stats, horizon)]
    recs = []
    for g in range(gens + 1):
        z = orc.noise(seed, g, 0, lam, st.n, stream=orc.STREAM_CMA_Z).astype(np.float32).astype(np.float64)
        X = st.ask(z)
        ret, osum, osq, cnt = po.rollouts(X.astype(np.float32), H, seed, g, np.arange(lam), reps, stats, horizon)
        cost = -ret.mean(1)
        tests.append(po.test_returns(X[int(np.argmin(cost))].astype(np.float32), H, seed, g + 1, reps, stats, horizon))
        if g == gens:
            break
        shaped = orc.fitness_shift(cost)
        st.tell(X, shaped)
        stats = po.merge_totals(stats, osum, osq, cnt)
        recs.append(dict(cost=cost, shaped=shaped, X=X, m=st.m.copy(), sigma=st.sigma, pc=st.pc.copy(), ps=st.ps.copy(),
                         C=st.C.copy(), stats=np.concatenate([stats[0], stats[1], [stats[2]]])))
        if stats_feed is not None:
            f = np.asarray(stats_feed[g], np.float32)
            stats = (f[:3], f[3:6], f[6])
    return recs, tests


def test_oracle_chain_matches_verbatim_reference_cma_train():
    g = np.load(GOLD)
    H, lam, reps, seed, gens = int(g['H']), int(g['lam']), int(g['reps']), int(g['seed']), int(g['gens'])
    assert (H, lam, reps, orc.param_count(3, H, 1)) == (16, 16, 10, 353)
    st = cma.CMAState(g['theta0'].astype(np.float64), 1.0, lam)
    assert st.gap == 4 > gens                                 # B = I, D = 1 throughout: no eigensolver enters
    assert list(g['train_steps']) == [k * lam * reps * po.HORIZON for k in range(gens + 2)]
    # Tolerances.  sigma = 1 solutions of a 16-unit net saturate: the torque is bang-bang at +-2, so a rounding-level
    # change in a pre-activation can flip one step's torque and move an episode's return by percents.  Before the first
    # merge (generation 0, test() calls 0 and 1) the fp64 oracle and the reference's fp32 torch agree to 1e-5.  Afterwards
    # the reference's statistics, accumulated one fp32 Welford step at a time, differ from exact sums by ~1e-5 and that is
    # amplified too.  Each generation therefore starts from the reference's own statistics (layered), and the later costs,
    # statistics and test means get bounds 1e-3, 2e-3 and 2e-2 (observed: 1.7e-4, 4.1e-4 and 9e-3).  Ranks, solutions and
    # the strategy state must agree to rounding in every generation.
    recs, tests = oracle_cma_chain(g['theta0'], H, lam, reps, seed, float(g['sigma']), gens, stats_feed=g['stats'])
    means = np.asarray([t.mean() for t in tests])
    assert np.allclose(means[:2], g['test_rewards'][:2], rtol=1e-5)
    assert np.allclose(means[2:], g['test_rewards'][2:], rtol=2e-2)
    for k, r in enumerate(recs):
        assert np.allclose(r['cost'], g['costs'][k], rtol=1e-5 if k == 0 else 1e-3)
        assert np.array_equal(r['shaped'], g['shaped'][k])                           # ranks (cma_es.py:89)
        assert np.max(np.abs(r['X'] - g['solutions'][k])) <= 1e-6 * np.max(np.abs(r['X']))
        assert np.allclose(r['stats'], g['stats'][k], rtol=2e-4 if k == 0 else 2e-3, atol=2e-5)
        assert np.max(np.abs(r['m'] - g['m'][k])) <= 1e-6 * np.max(np.abs(g['m'][k]))
        assert abs(r['sigma'] - float(g['sigmas'][k])) <= 1e-12
        assert np.max(np.abs(r['pc'] - g['pc'][k])) <= 1e-6 * np.max(np.abs(g['pc'][k]))
        assert np.max(np.abs(r['ps'] - g['ps'][k])) <= 1e-6 * np.max(np.abs(g['ps'][k]))


def _train_worker():
    from distributedes_b200 import cma_es
    from distributedes_b200.config import ClosedLoopPendulumConfig
    g = np.load(GOLD)
    cfg = ClosedLoopPendulumConfig(16)
    cfg.initial_weight = g['theta0'].copy()
    cfg.pop_size, cfg.sigma, cfg.seed = int(g['lam']), float(g['sigma']), int(g['seed'])
    cfg.max_steps = (int(g['gens']) + 1) * cfg.pop_size * cfg.repetitions * 200 - 1
    worker = cma_es.Worker(dist.get_rank(), None, None, None, None, cfg, device='cpu', kernels=cpu_ops)
    es = cma_es.CMAEvolutionStrategy(cfg.initial_weight, cfg.sigma, cfg.pop_size, seed=cfg.seed, device='cpu',
                                     kernels=cpu_ops)
    told = []
    real_tell = es.tell

    def spy_tell(solutions, cost):
        told.append(np.asarray(cost, dtype=np.float64).copy())
        return real_tell(solutions, cost)
    es.tell = spy_tell
    rewards, steps, stamps = cma_es.train(cfg, worker=worker, es=es)
    return dict(rewards=np.asarray(rewards), steps=np.asarray(steps), n_stamps=len(stamps), m=es.m.numpy(),
                C=es.C.numpy(), sigma=es.sigma, pc=es.pc.numpy(), stats=worker.obs_stats.numpy(), shaped=np.stack(told),
                n_local=es.n_local)


@pytest.mark.parametrize('world', [2, 3])
def test_cma_train_closed_loop_sharded_packed_reproduces_the_reference_golden(world):
    """cma_es.train(ClosedLoopPendulumConfig(16)) on gloo ranks (8 + 8 members, and the ragged 6 + 5 + 5): every rank returns
    the same triple and holds the same strategy state, equal to the reference's verbatim run.  tell() all-reduces the
    rank-mu partials in the packed form sharded GPU runs use."""
    g = np.load(GOLD)
    r = spawn(world, _train_worker)
    assert sum(int(x['n_local']) for x in r) == int(g['lam'])
    for x in r[1:]:
        for k in ('rewards', 'steps', 'm', 'C', 'sigma', 'pc', 'stats', 'shaped'):
            assert np.array_equal(r[0][k], x[k]), k
    assert list(r[0]['steps']) == list(g['train_steps']) and int(r[0]['n_stamps']) == len(g['train_steps'])
    # not layered: the statistics are the chain's own (tolerances: see the oracle test above; observed 1.6e-2, 2.6e-3)
    assert np.allclose(r[0]['rewards'][:2], g['test_rewards'][:2], rtol=1e-5)
    assert np.allclose(r[0]['rewards'][2:], g['test_rewards'][2:], rtol=3e-2)
    assert np.array_equal(r[0]['shaped'], g['shaped'].astype(np.float32).astype(np.float64))
    assert np.allclose(r[0]['stats'], g['stats'][-1], rtol=5e-3, atol=2e-5)
    # strategy state: fp32 C and sampling against the fp64 restatement fed the reference's own solutions and ranks
    ref = cma.CMAState(g['theta0'].astype(np.float64), float(g['sigma']), int(g['lam']))
    for k in range(int(g['gens'])):
        ref.tell(g['solutions'][k].astype(np.float64), g['shaped'][k])
    assert np.max(np.abs(ref.m - g['m'][-1])) <= 1e-6 * np.max(np.abs(g['m'][-1]))
    assert np.linalg.norm(r[0]['m'] - g['m'][-1]) <= 2e-5 * np.linalg.norm(g['m'][-1])
    assert np.linalg.norm(r[0]['pc'] - g['pc'][-1]) <= 2e-5 * np.linalg.norm(g['pc'][-1])
    assert abs(float(r[0]['sigma']) - float(g['sigmas'][-1])) <= 2e-5 * float(g['sigmas'][-1])
    assert np.linalg.norm(r[0]['C'] - ref.C) <= 2e-5 * np.linalg.norm(ref.C)


def test_hidden_16_is_accepted_on_the_closed_loop_path():
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(16)
    assert (c.hidden_size, len(c.initial_weight), c.repetitions) == (16, 353, 10)
    assert ClosedLoopPendulumConfig().hidden_size == 64
    with pytest.raises(ValueError, match='hidden_size'):
        ClosedLoopPendulumConfig(48)


def test_rollout_eval_solutions_validates_before_cuda(lib):
    import ctypes as C
    from distributedes_b200 import _lib
    d = _lib.Dims(3, 16, 1, 200)
    buf = (C.c_float * 16)()
    args = lambda env=0, dims=d, reps=10, ws=None, ws_bytes=0, n=4, ptr=None, totals=None: (
        ptr, None, totals, ptr, None, env, dims, reps, 2.0, 0.0, 0, 0, 0, n, ws, ws_bytes, None)
    assert lib.des_rollout_eval_solutions(*args(env=7)) == -1 and b'unknown environment' in lib.des_last_error()
    assert lib.des_rollout_eval_solutions(*args(dims=_lib.Dims(3, 48, 1, 200))) == -1
    assert b'multiple of 32' in lib.des_last_error() and b'des_rollout_eval_solutions' in lib.des_last_error()
    assert lib.des_rollout_eval_solutions(*args(reps=11)) == -1 and b'repetitions' in lib.des_last_error()
    assert lib.des_rollout_eval_solutions(*args()) == -1 and b'NULL' in lib.des_last_error()
    # obs totals need n_local * 7 doubles of workspace
    rc = lib.des_rollout_eval_solutions(*args(ptr=C.cast(buf, C.c_void_p), totals=C.cast(buf, C.c_void_p),
                                              ws=C.cast(buf, C.c_void_p), ws_bytes=64))
    assert rc == -4 and b'workspace' in lib.des_last_error()
    assert lib.des_rollout_eval_solutions(*args(n=0)) == 0
    # des_rollout_eval takes H = 16 too, and still rejects 48
    rc = lib.des_rollout_eval(None, None, None, None, None, 0, d, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, 4, 0, None, 0, None)
    assert rc == -1 and b'NULL' in lib.des_last_error()
