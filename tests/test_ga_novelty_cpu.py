"""The genetic algorithm's novelty search without a GPU, over the stand-ins (tests/cpu_ops.py, cpu_ops_ga.py,
cpu_ops_novelty.py and cpu_ops_ga_novelty.py):

  - the oracle's order at w = 1 is ga_oracle.order, ties, NaN, +-0 and +-inf included, and at w = 0 the order of the
    novelty, descending; in between it is the contract's keys, sorted;
  - novelty.train_ga at w = 0, 0.5 and 'adaptive' equals tests/ga_novelty_oracle.py's chain, closed-loop and
    host-stepped: rewards, steps, the archive in order, the weights, every selection's inputs and the final table;
  - at w = 1 it is genetic.train, bit for bit (rewards, steps, final table, order, statistics);
  - the archive buffer, the GA tell with novelty, and every refusal, before any device work.
"""
import types

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import cpu_ops  # noqa: E402
import cpu_ops_ga  # noqa: E402
import cpu_ops_ga_novelty  # noqa: E402
import cpu_ops_novelty  # noqa: E402
import ga_novelty_oracle as gno  # noqa: E402
from host_env_support import PendulumProbe  # noqa: E402
from oracle import ga_oracle as gao  # noqa: E402
from oracle import nes_oracle as orc  # noqa: E402
from oracle import novelty_oracle as no  # noqa: E402
from oracle import pendulum_oracle as po  # noqa: E402

H = 16
HORIZON = 6
K = types.SimpleNamespace(**{k: v for m in (cpu_ops, cpu_ops_ga, cpu_ops_novelty, cpu_ops_ga_novelty)
                             for k, v in vars(m).items() if not k.startswith('_') and callable(v)})


@pytest.fixture(autouse=True)
def _clear():
    for m in (cpu_ops_ga, cpu_ops_novelty, cpu_ops_ga_novelty):
        m.CALLS.clear()


# ---- the oracle's order ----------------------------------------------------------------------------------------------
SPECIAL = np.array([1.0, np.nan, -0.0, 3.0, 0.0, 3.0, -np.inf, np.nan, 2.0, np.inf, -1.0, 0.0], dtype=np.float32)


def test_the_order_at_weight_1_is_the_fitness_order():
    rs = np.random.RandomState(0)
    for f in (SPECIAL, np.round(rs.randn(300), 1).astype(np.float32)):
        nov = rs.permutation(np.concatenate([SPECIAL, rs.randn(f.size)]))[:f.size].astype(np.float32)
        for T in (1, 3, f.size):
            assert gno.ns_ga_order(f, nov, 1.0, T).tolist() == gao.order(f, T).tolist()


def test_the_order_at_weight_0_is_the_novelty_order():
    rs = np.random.RandomState(1)
    for nov in (SPECIAL, np.round(rs.randn(300), 1).astype(np.float32)):
        f = rs.randn(nov.size).astype(np.float32)
        for T in (1, 5, nov.size):
            assert gno.ns_ga_order(f, nov, 0.0, T).tolist() == gao.order(nov, T).tolist()


def test_nan_fitness_and_nan_novelty_rank_worst_in_their_own_term():
    f = np.array([np.nan, 1.0, 2.0, 3.0], dtype=np.float32)
    nov = np.array([5.0, 1.0, 2.0, np.nan], dtype=np.float32)
    # c_f = (0.5, 1/6, -1/6, -0.5) and c_n = (-0.5, 1/6, -1/6, 0.5): member 0 is the most novel with the worst (NaN)
    # fitness, member 3 the fittest with the worst (NaN) novelty.  At w = 0.5 both keys are 0, a tie to index 0, behind
    # member 2's -1/6; at w = 0.3 member 0 leads (-0.2) and member 3 trails (0.2).
    assert gno.ns_ga_order(f, nov, 0.5, 4).tolist() == [2, 0, 3, 1]
    assert gno.ns_ga_order(f, nov, 0.3, 4).tolist() == [0, 2, 1, 3]


def test_the_keys_are_the_contract_s():
    rs = np.random.RandomState(2)
    f, nov = rs.randn(50).astype(np.float32), np.abs(rs.randn(50)).astype(np.float32)
    for w in (0.0, 0.3, 0.5, 1.0):
        c_f = (orc.ranks_stable(-f) / 49.0 - 0.5).astype(np.float32)
        c_n = (orc.ranks_stable(-nov) / 49.0 - 0.5).astype(np.float32)
        key = no.fmaf32(np.float32(w), c_f, np.float32(1.0 - w) * c_n)
        assert gno.keys(f, nov, w).tobytes() == key.tobytes()
        assert gno.ns_ga_order(f, nov, w, 50).tolist() == sorted(range(50), key=lambda i: (key[i], i))


# ---- train_ga over the stand-ins -------------------------------------------------------------------------------------
# Closed-loop runs are without action noise: the stand-ins of test episodes differ there (cpu_ops.rollout_eval draws none,
# cpu_ops_novelty.rollout_eval_bc draws it as the test member's), so w = 1 could not be compared with genetic.train.
# The GPU tests run the fused kernel with action noise on.
def _closed(N=6, T=3, E=1, gens=4, w=0.5, noise=0.0):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(H)
    c.pop_size, c.truncation, c.elites, c.max_generations, c.seed, c.sigma = N, T, E, gens, 5, 0.05
    c.repetitions = c.test_repetitions = 2
    c.action_noise_std = noise
    c.initial_weight = orc.synthetic_theta(3, H, 1, seed=1)
    c.ns_reward_weight, c.ns_k = w, 3
    return c


def _host(N=6, T=3, E=1, gens=3, w=0.5):
    from distributedes_b200.config import HostEnvConfig
    c = HostEnvConfig(PendulumProbe, hidden_size=H, clip=2.0, batch_env_fn=lambda B: po.PendulumBatch(B, 5, HORIZON))
    c.pop_size, c.truncation, c.elites, c.max_generations, c.seed, c.sigma = N, T, E, gens, 5, 0.05
    c.repetitions = c.test_repetitions = 2
    c.initial_weight = orc.synthetic_theta(3, H, 1, seed=1)
    c.ns_reward_weight, c.ns_k = w, 3
    return c


def _nsga(c):
    from distributedes_b200 import novelty
    nsga = novelty.build_ga(c, kernels=K, device='cpu')
    if hasattr(nsga.worker.source, 'horizon'):
        nsga.worker.source.horizon = nsga.worker.source.T = HORIZON
    return nsga


def _chain(c, host):
    N, reps = c.pop_size, c.repetitions
    zero = (np.zeros(3, np.float32), np.zeros(3, np.float32), np.float32(0))
    st = dict(stats=zero, totals=None)

    def episodes(rows, g, members, n_reps, noise_offset):
        env = no.FinalObs(po.PendulumBatch(len(members) * n_reps, c.seed, HORIZON), 3)
        ret, n, totals = po.episodes(rows, env, 3, H, 1, c.clip, g, members, n_reps, st['stats'], c.seed, noise_offset,
                                     c.action_noise_std)
        return ret, n, totals, no.behaviours(env.final, len(members), n_reps)

    def evaluate(rows, g):
        ret, n, totals, bc = episodes(rows, g, np.arange(N), reps, 0)
        st['totals'] = totals
        return ret.mean(1).astype(np.float32), bc, (n if host else N * reps * HORIZON)

    def test(theta, k):
        ret, _, _, bc = episodes(theta[None], k, [po.TEST_MEMBER], c.test_repetitions, 0)
        return (ret[0] if host else ret[0].astype(np.float32).astype(np.float64)), bc[0]

    def merge(g):
        st['stats'] = po.merge_totals(st['stats'], *st['totals'])
    return gno.train(c.initial_weight, sigma=c.sigma, N=N, T=c.truncation, E=c.elites, seed=c.seed, k=c.ns_k,
                     w=c.ns_reward_weight, generations=c.max_generations, evaluate=evaluate, test=test, merge=merge)


@pytest.mark.parametrize('kind', ['closed', 'host'])
@pytest.mark.parametrize('w', [0.0, 0.5, 'adaptive'])
def test_train_ga_follows_the_oracle_chain(kind, w):
    from distributedes_b200 import novelty
    c = (_closed if kind == 'closed' else _host)(w=w)
    nsga = _nsga(c)
    rewards, steps, _ = novelty.train_ga(c, nsga)
    chain = _chain(c, kind == 'host')
    assert rewards == chain['rewards'] and steps == chain['steps']
    assert nsga.archive.numpy().tobytes() == chain['archive'].tobytes()
    assert nsga.archive.shape == (1 + c.max_generations, 3)
    assert nsga.weights == chain['weights']
    assert nsga.ga.parents.numpy().tobytes() == chain['tables'][-1].tobytes()
    assert nsga.ga.order.numpy().tolist() == chain['orders'][-1].tolist()
    orders = [x for x in cpu_ops_ga_novelty.CALLS if x['op'] == 'ns_ga_order']
    assert len(orders) == c.max_generations
    for x, f, nov, wg in zip(orders, chain['fitness'], chain['novelty'], chain['weights']):
        assert x['fitness'].numpy().tobytes() == f.tobytes()
        assert x['novelty'].numpy().tobytes() == nov.tobytes()
        assert (x['reward_weight'], x['truncation']) == (wg, c.truncation)
    if kind == 'closed':
        assert [x['op'] for x in cpu_ops_ga_novelty.CALLS if x['op'] == 'rollout_eval_ga_bc'] == \
            ['rollout_eval_ga_bc'] * c.max_generations
        assert [x['op'] for x in cpu_ops_ga.CALLS if x['op'] in ('rollout_eval_ga', 'ga_order')] == []
        assert [x['op'] for x in cpu_ops_novelty.CALLS if x['op'] == 'rollout_eval_bc'] == \
            ['rollout_eval_bc'] * (1 + c.max_generations)


def test_the_schedule_is_nsra_es_s():
    nsga = _nsga(_closed(w='adaptive'))
    rs = np.random.RandomState(4)
    w, stall = 1.0, 0
    for improved in rs.rand(200) < 0.1:
        nsga.adapt(bool(improved))
        w, stall = no.adapt(w, stall, bool(improved))
        assert (nsga.reward_weight, nsga.stall) == (w, stall)
    assert w < 1.0                                                       # the sequence does lower it
    fixed = _nsga(_closed(w=0.5))
    for _ in range(20):
        fixed.adapt(False)
    assert fixed.reward_weight == 0.5


@pytest.mark.parametrize('kind', ['closed', 'host'])
def test_train_ga_at_weight_1_is_genetic_train(kind):
    from distributedes_b200 import genetic, novelty
    c = (_closed if kind == 'closed' else _host)(w=1.0)
    worker, ga = genetic.build(c, kernels=K, device='cpu')
    if hasattr(worker.source, 'horizon'):
        worker.source.horizon = worker.source.T = HORIZON
    want = genetic.train(c, worker, ga)
    nsga = _nsga(c)
    got = novelty.train_ga(c, nsga)
    assert got[0] == want[0] and got[1] == want[1]
    assert nsga.ga.parents.numpy().tobytes() == ga.parents.numpy().tobytes()
    assert nsga.ga.order.numpy().tobytes() == ga.order.numpy().tobytes()
    if worker.obs_stats is not None:
        assert nsga.worker.obs_stats.numpy().tobytes() == worker.obs_stats.numpy().tobytes()
    assert nsga.weights == [1.0] * c.max_generations


def test_host_stepped_ga_behaviours_are_the_final_observations_averaged():
    c = _host()
    nsga = _nsga(c)
    fit = nsga.evaluate()
    rows = gao.member_rows(np.asarray(c.initial_weight, np.float32)[None], 1, c.sigma, c.seed, 0, np.arange(6))   # E_0 = 1
    env = no.FinalObs(po.PendulumBatch(6 * 2, 5, HORIZON), 3)
    ret, _, _ = po.episodes(rows, env, 3, H, 1, c.clip, 0, np.arange(6), 2, None, c.seed)
    assert nsga.bc.numpy().tobytes() == no.behaviours(env.final, 6, 2).tobytes()
    assert fit.numpy().tobytes() == ret.mean(1).astype(np.float32).tobytes()


def test_tell_with_novelty_orders_by_the_blend_and_gathers_as_without():
    from distributedes_b200 import genetic
    ga = genetic.GeneticAlgorithm(orc.synthetic_theta(3, H, 1, seed=1), 0.1, 8, truncation=4, elites=2, device='cpu',
                                  kernels=K)
    rs = np.random.RandomState(3)
    f, nov = rs.randn(8).astype(np.float32), rs.rand(8).astype(np.float32)
    rows = ga.ask().numpy()
    order = ga.tell(torch.from_numpy(f), torch.from_numpy(nov), 0.25)
    want = gno.ns_ga_order(f, nov, 0.25, 4)
    assert order.numpy().tolist() == want.tolist()
    assert ga.parents.numpy().tobytes() == rows[want].tobytes()
    with pytest.raises(ValueError, match='novelty of all 8 members \\(got 7\\)'):
        ga.tell(torch.from_numpy(f), torch.zeros(7), 0.5)


def test_the_archive_doubles_when_full():
    from distributedes_b200 import novelty
    store = novelty.Archive(3, 'cpu')
    cap = store.buffer.shape[0]
    rows = torch.arange(3 * (cap + 5), dtype=torch.float32).reshape(-1, 3)
    for r in rows:
        store.add(r)
    assert store.buffer.shape[0] == 2 * cap and store.size == cap + 5
    assert torch.equal(store.rows, rows)


def test_test_ga_is_genetic_test():
    from distributedes_b200 import genetic, novelty
    c = _closed()
    nsga = _nsga(c)
    worker, _ = genetic.build(c, kernels=K, device='cpu')
    worker.source.horizon = worker.source.T = HORIZON
    assert novelty.test_ga(c, c.initial_weight, None, nsga) == genetic.test(c, c.initial_weight, None, worker)


# ---- refusals --------------------------------------------------------------------------------------------------------
def _no_device_work():
    return cpu_ops_ga.CALLS == [] and cpu_ops_novelty.CALLS == [] and cpu_ops_ga_novelty.CALLS == []


@pytest.mark.parametrize('change,match', [
    (dict(mirrored=True), 'mirrored sampling'),
    (dict(ns_agents=2), 'ns_agents = 2; the genetic algorithm evolves one population'),
    (dict(ns_agents=0), 'ns_agents must be >= 1'),
    (dict(ns_k=0), 'ns_k 0 is not in'),
    (dict(ns_k=33), 'ns_k 33 is not in'),
    (dict(ns_reward_weight=1.5), 'ns_reward_weight 1.5 is not in'),
    (dict(ns_reward_weight='adapt'), "or 'adaptive'"),
    (dict(state_dim=33), 'state_dim = 33'),
    (dict(state_dim=0), 'state_dim = 0'),
    (dict(pop_size=1), 'pop_size 1 < 2'),
    (dict(truncation=0), 'truncation 0 is not in \\[1, pop_size = 6\\]'),
    (dict(truncation=7), 'truncation 7 is not in \\[1, pop_size = 6\\]'),
    (dict(elites=4), 'elites 4 is not in \\[0, truncation = 3\\]'),
])
def test_refusals(change, match):
    from distributedes_b200 import novelty
    c = _closed()
    for k, v in change.items():
        setattr(c, k, v)
    for call in (lambda: novelty.train_ga(c), lambda: novelty.build_ga(c, kernels=K, device='cpu'),
                 lambda: novelty.check_ga_config(c)):
        with pytest.raises(ValueError, match=match):
            call()
    assert _no_device_work()


def test_tape_configs_are_refused():
    from distributedes_b200 import novelty
    from distributedes_b200.config import PendulumConfig
    with pytest.raises(ValueError, match='a tape has no episodes'):
        novelty.train_ga(PendulumConfig(H))
    assert _no_device_work()


def test_several_ranks_are_refused(monkeypatch):
    from distributedes_b200 import novelty
    monkeypatch.setattr(novelty.dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(novelty.dist, 'get_world_size', lambda *a: 2)
    with pytest.raises(ValueError, match='one process; the process group has world size 2'):
        novelty.train_ga(_closed())
    assert _no_device_work()
