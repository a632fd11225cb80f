"""Novelty search without a GPU, over the stand-ins (tests/cpu_ops.py with tests/cpu_ops_novelty.py):

  - novelty.train with one agent and reward weight 1 is natural_es.train, bit for bit (rewards, steps, final theta), on
    the closed-loop Pendulum and on a host-stepped Pendulum;
  - with three agents it is oracle/novelty_oracle.py's chain for w = 0, 0.5 and 'adaptive': rewards, steps, archive rows
    in order, agent selections and the weight of every generation;
  - the NSRA-ES schedule, host-stepped behaviours, the archive's growth, and every refusal.
"""
import types

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import cpu_ops
import cpu_ops_novelty
from host_env_support import PendulumProbe
from oracle import nes_oracle as orc
from oracle import novelty_oracle as no
from oracle import pendulum_oracle as po

H = 16
HORIZON = 6
K = types.SimpleNamespace(**{k: v for m in (cpu_ops, cpu_ops_novelty) for k, v in vars(m).items()
                             if not k.startswith('_') and callable(v)})


@pytest.fixture(autouse=True)
def _clear():
    cpu_ops_novelty.CALLS.clear()


def _closed(N=6, gens=3, w=1.0, M=1, k=3):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(H)
    c.pop_size, c.max_generations, c.seed, c.sigma, c.learning_rate = N, gens, 5, 0.05, 0.05
    c.repetitions = c.test_repetitions = 2
    c.initial_weight = orc.synthetic_theta(3, H, 1, seed=1)
    c.ns_reward_weight, c.ns_agents, c.ns_k = w, M, k
    return c


def _host(N=6, gens=3, w=1.0, M=1):
    from distributedes_b200.config import HostEnvConfig
    c = HostEnvConfig(PendulumProbe, hidden_size=H, clip=2.0, batch_env_fn=lambda B: po.PendulumBatch(B, 5, HORIZON))
    c.pop_size, c.max_generations, c.seed, c.sigma, c.learning_rate = N, gens, 5, 0.05, 0.05
    c.repetitions = c.test_repetitions = 2
    c.initial_weight = orc.synthetic_theta(3, H, 1, seed=1)
    c.ns_reward_weight, c.ns_agents = w, M
    return c


def _short(engine):
    if hasattr(engine.source, 'horizon'):
        engine.source.horizon = engine.source.T = HORIZON


def _ns(c):
    from distributedes_b200 import novelty
    ns = novelty.build(c, kernels=K, device='cpu')
    for e in ns.agents:
        _short(e)
    return ns


@pytest.mark.parametrize('kind', ['closed', 'host'])
def test_one_agent_at_weight_1_is_natural_es(kind):
    from distributedes_b200 import natural_es, novelty
    c = (_closed if kind == 'closed' else _host)()
    engine = natural_es.build_engine(c, kernels=K, device='cpu')
    _short(engine)
    want = natural_es.train(c, engine)
    ns = _ns(c)
    got = novelty.train(c, ns)
    assert got[0] == want[0] and got[1] == want[1]
    assert ns.agents[0].theta.numpy().tobytes() == engine.theta.numpy().tobytes()
    assert ns.selected == [0] * 4 and ns.weights == [1.0] * 3
    assert ns.archive.shape == (4, 3)
    if kind == 'closed':
        assert [x['op'] for x in cpu_ops_novelty.CALLS if x['op'] == 'rollout_eval_bc'] == ['rollout_eval_bc'] * 8


def _chain(c, gens):
    from distributedes_b200.model import StandardFCNet
    M, N, reps = c.ns_agents, c.pop_size, c.repetitions
    seeds = [c.seed + m for m in range(M)]
    thetas = [c.initial_weight] + [StandardFCNet(3, 1, H, seed=m).get_weight() for m in range(1, M)]
    zero = (np.zeros(3, np.float32), np.zeros(3, np.float32), np.float32(0))
    st = dict(stats=[zero] * M, totals=[None] * M)

    def evaluate(m, rows, g):
        ret, totals, bc = no.closed_episodes(rows, H, seeds[m], g, np.arange(N), reps, st['stats'][m], HORIZON, c.clip)
        st['totals'][m] = totals
        return ret.mean(1).astype(np.float32), bc, N * reps * HORIZON

    def test(m, theta, g):
        ret, _, bc = no.closed_episodes(theta[None], H, seeds[m], g, [po.TEST_MEMBER], c.test_repetitions,
                                        st['stats'][m], HORIZON, c.clip)
        return ret[0].astype(np.float32).astype(np.float64), bc[0]

    def merge(m):
        st['stats'][m] = po.merge_totals(st['stats'][m], *st['totals'][m])
    return no.train(thetas, N=N, sigma=c.sigma, lr=c.learning_rate, wd=c.weight_decay, seeds=seeds, k=c.ns_k,
                    w=c.ns_reward_weight, generations=gens, evaluate=evaluate, test=test, merge=merge, rng_seed=c.seed)


@pytest.mark.parametrize('w', [0.0, 0.5, 'adaptive'])
def test_three_agents_follow_the_oracle_chain(w):
    from distributedes_b200 import novelty
    gens = 5
    c = _closed(gens=gens, w=w, M=3)
    ns = _ns(c)
    rewards, steps, _ = novelty.train(c, ns)
    chain = _chain(c, gens)
    assert rewards == chain['rewards'] and steps == chain['steps']
    assert ns.selected == chain['selected'] and ns.weights == chain['weights']
    assert ns.archive.numpy().tobytes() == chain['archive'].tobytes()
    assert ns.archive.shape == (3 + gens, 3)
    for e, theta in zip(ns.agents, chain['thetas']):
        assert e.theta.numpy().tobytes() == theta.tobytes()
    shapes = [x['reward_weight'] for x in cpu_ops_novelty.CALLS if x['op'] == 'ns_shape']
    assert shapes == chain['weights']


def test_the_trainer_s_schedule_is_the_oracle_s():
    ns = _ns(_closed(w='adaptive'))
    rs = np.random.RandomState(4)
    w, stall = 1.0, 0
    for improved in rs.rand(200) < 0.1:
        ns.adapt(bool(improved))
        w, stall = no.adapt(w, stall, bool(improved))
        assert (ns.reward_weight, ns.stall) == (w, stall)
    assert w < 1.0                                                       # the sequence does lower it


def test_a_fixed_weight_does_not_adapt():
    ns = _ns(_closed(w=0.5))
    for _ in range(20):
        ns.adapt(False)
    assert ns.reward_weight == 0.5


def test_host_stepped_behaviours_are_the_final_observations_averaged():
    c = _host()
    ns = _ns(c)
    e = ns.agents[0]
    fit = e.evaluate(bc_out=ns.bc)
    rows = orc.perturb(c.initial_weight, c.sigma, orc.noise(c.seed, 0, 0, c.pop_size, e.P))
    env = no.FinalObs(po.PendulumBatch(c.pop_size * 2, 5, HORIZON), 3)
    ret, _, _ = po.episodes(rows, env, 3, H, 1, c.clip, 0, np.arange(c.pop_size), 2, None, c.seed)
    np.testing.assert_array_equal(ns.bc.numpy(), no.behaviours(env.final, c.pop_size, 2))
    np.testing.assert_array_equal(fit.numpy(), ret.mean(1).astype(np.float32))


def test_mirrored_device_members_have_no_behaviours():
    from distributedes_b200 import natural_es
    c = _closed()
    c.mirrored = True
    engine = natural_es.build_engine(c, kernels=K, device='cpu')
    with pytest.raises(ValueError, match='plain members only'):
        engine.evaluate(bc_out=torch.zeros((c.pop_size, 3)))
    assert cpu_ops_novelty.CALLS == []


def test_the_archive_doubles_when_full():
    ns = _ns(_closed())
    cap = ns._archive.shape[0]
    rows = torch.arange(3 * (cap + 5), dtype=torch.float32).reshape(-1, 3)
    for r in rows:
        ns._archive_add(r)
    assert ns._archive.shape[0] == 2 * cap and ns.size == cap + 5
    assert torch.equal(ns.archive, rows)


def test_the_selection_draw():
    rng_a, rng_b = (np.random.Generator(np.random.PCG64(3)) for _ in range(2))
    nov = np.array([np.nan, 0.0, 2.0, 1.0], dtype=np.float32)
    draws = [no.select(rng_a, nov) for _ in range(200)]
    assert set(draws) == {2, 3}
    assert [no.select(rng_b, np.zeros(4, np.float32)) for _ in range(200)].count(0) > 20      # uniform


@pytest.mark.parametrize('setup,match', [
    (lambda c: setattr(c, 'mirrored', True), 'mirrored sampling'),
    (lambda c: setattr(c, 'ns_k', 0), 'ns_k 0 is not in'),
    (lambda c: setattr(c, 'ns_k', 33), 'ns_k 33 is not in'),
    (lambda c: setattr(c, 'ns_agents', 0), 'ns_agents must be >= 1'),
    (lambda c: setattr(c, 'ns_reward_weight', 1.5), 'ns_reward_weight 1.5 is not in'),
    (lambda c: setattr(c, 'ns_reward_weight', -0.1), 'is not in \\[0, 1\\]'),
    (lambda c: setattr(c, 'ns_reward_weight', 'adapt'), "or 'adaptive'"),
    (lambda c: setattr(c, 'state_dim', 33), 'state_dim = 33'),
])
def test_refusals(setup, match):
    from distributedes_b200 import novelty
    c = _closed()
    setup(c)
    with pytest.raises(ValueError, match=match):
        novelty.train(c)
    with pytest.raises(ValueError, match=match):
        novelty.build(c, kernels=K, device='cpu')
    assert cpu_ops_novelty.CALLS == []


def test_tape_configs_are_refused():
    from distributedes_b200 import novelty
    from distributedes_b200.config import PendulumConfig
    with pytest.raises(ValueError, match='a tape has no episodes'):
        novelty.train(PendulumConfig())


def test_several_ranks_are_refused(monkeypatch):
    from distributedes_b200 import novelty
    monkeypatch.setattr(novelty.dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(novelty.dist, 'get_world_size', lambda *a: 2)
    with pytest.raises(ValueError, match='one process; the process group has world size 2'):
        novelty.train(_closed())
