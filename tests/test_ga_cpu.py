"""The genetic algorithm without a GPU:

  - des_ga_rows, des_rollout_eval_ga and des_ga_order refuse bad arguments before any CUDA work (des_rollout_eval_ga
    also everything des_rollout_eval refuses, with its message under its own name); n_local = 0 does nothing;
  - the wrappers check their tensors in ops._ptr;
  - the oracle's parent draws equal a scalar restatement of Philox4x32-7 word for word, and its order is the contract's;
  - genetic.train over tests/cpu_ops_ga.py equals oracle/ga_oracle.py's chain: closed-loop (fused and materialised
    rows), tape and host-stepped SynthWalk;
  - the refusals: mirrored sampling, several ranks, N < 2, truncation and elites out of range.
"""
import ctypes as C
import types

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import cpu_ops
import cpu_ops_ga
from lib_fixture import lib  # noqa: F401
from oracle import ga_oracle as gao
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from oracle.synth_walk import SynthWalkEnv

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work
H = 16
P = orc.param_count(3, H, 1)


def _msg(lib):
    return lib.des_last_error().decode()


# ---- the entry points ------------------------------------------------------------------------------------------------
# case -> (n_parents, n_elites, P, member_offset, n_local, null, expected message)
ROWS = {
    'n_local_negative': (2, 0, 9, 0, -1, False, 'des_ga_rows: bad size (n_local=-1, P=9)'),
    'P_0': (2, 0, 0, 0, 2, False, 'des_ga_rows: bad size (n_local=2, P=0)'),
    'n_parents_0': (0, 0, 9, 0, 2, False, 'des_ga_rows: n_parents must be in [1, 2^31) (got 0)'),
    'elites_negative': (2, -1, 9, 0, 2, False, 'des_ga_rows: n_elites must be in [0, n_parents = 2] (got -1)'),
    'elites_past_parents': (2, 3, 9, 0, 2, False, 'des_ga_rows: n_elites must be in [0, n_parents = 2] (got 3)'),
    'past_2^32': (2, 0, 9, (1 << 32) - 1, 2, False, 'des_ga_rows: member index must fit 32 bits'),
    'null': (2, 0, 9, 0, 2, True, 'des_ga_rows: NULL pointer'),
}


@pytest.mark.parametrize('case', list(ROWS))
def test_ga_rows_refuses(lib, case):  # noqa: F811
    n_parents, n_elites, p, off, n, null, msg = ROWS[case]
    rc = lib.des_ga_rows(None if null else D, None if null else C.c_void_p(1 << 20), n_parents, n_elites, p, 0.1, 0, 0,
                         off, n, None, None)
    assert rc == -1 and _msg(lib) == msg


def test_ga_rows_refuses_rows_that_overlap_the_parents(lib):  # noqa: F811
    base = 1 << 20
    for out in (base, base + 4 * 9, base - 4 * 9 * 2 + 4):        # the same rows, the second row, the tail of rows_out
        rc = lib.des_ga_rows(C.c_void_p(out), C.c_void_p(base), 2, 0, 9, 0.1, 0, 0, 0, 2, None, None)
        assert rc == -1 and _msg(lib) == 'des_ga_rows: rows_out overlaps parents (the table is double-buffered)'
    assert lib.des_ga_rows(None, None, 1, 0, 9, 0.1, 0, 0, 0, 0, None, None) == 0      # n_local == 0: nothing


# the cases of des_rollout_eval that des_rollout_eval_ga shares: (env, H, repetitions, tape_len, member_offset, n_local,
# null pointers, workspace bytes with totals requested or None)
EVAL = {
    'bad_env': (1, 32, 10, 200, 0, 2, False, None),
    'bad_width': (0, 48, 10, 200, 0, 2, False, None),
    'reps_0': (0, 32, 0, 200, 0, 2, False, None),
    'reps_11': (0, 32, 11, 200, 0, 2, False, None),
    'tape_0': (0, 32, 10, 0, 0, 2, False, None),
    'neg_offset': (0, 32, 10, 200, -2, 2, False, None),
    'past_2^28': (0, 32, 10, 200, (1 << 28) - 2, 4, False, None),
    'null_count': (0, 32, 10, 200, 0, 2, True, None),
    'small_workspace': (0, 32, 10, 200, 0, 2, False, 8),
}


@pytest.mark.parametrize('case', list(EVAL))
def test_rollout_eval_ga_refuses_what_des_rollout_eval_refuses(lib, case):  # noqa: F811
    from distributedes_b200 import _lib
    env, h, reps, T, off, n, null, ws = EVAL[case]
    p, tot, dims = None if null else D, None if ws is None else D, _lib.Dims(3, h, 1, T)
    wsp = None if ws is None else D
    rc = lib.des_rollout_eval(p, None, tot, p, None, env, dims, reps, 0.1, 2.0, 0.0, 0, 0, None, off, n, 0, wsp, ws or 0,
                              None)
    ev = (rc, _msg(lib))
    rc = lib.des_rollout_eval_ga(p, None, tot, p, 2, 1, None, env, dims, reps, 0.1, 2.0, 0.0, 0, 0, None, off, n, 0, wsp,
                                 ws or 0, None)
    assert ev[0] != 0 and rc == ev[0]
    assert _msg(lib) == ev[1].replace('des_rollout_eval', 'des_rollout_eval_ga', 1)


@pytest.mark.parametrize('n_parents,n_elites,noiseless,msg', [
    (2, 0, 1, 'des_rollout_eval_ga: test episodes (noiseless) evaluate one row; use des_rollout_eval on it'),
    (0, 0, 0, 'des_rollout_eval_ga: n_parents must be in [1, 2^31) (got 0)'),
    (2, 3, 0, 'des_rollout_eval_ga: n_elites must be in [0, n_parents = 2] (got 3)'),
    (2, -1, 0, 'des_rollout_eval_ga: n_elites must be in [0, n_parents = 2] (got -1)'),
])
def test_rollout_eval_ga_refuses_its_own(lib, n_parents, n_elites, noiseless, msg):  # noqa: F811
    from distributedes_b200 import _lib
    rc = lib.des_rollout_eval_ga(D, None, None, D, n_parents, n_elites, None, 0, _lib.Dims(3, 16, 1, 200), 10, 0.1, 2.0,
                                 0.0, 0, 0, None, 0, 2, noiseless, None, 0, None)
    assert rc == -1 and _msg(lib) == msg
    assert lib.des_rollout_eval_ga(None, None, None, None, 1, 0, None, 0, _lib.Dims(3, 16, 1, 200), 10, 0.1, 2.0, 0.0, 0,
                                   0, None, 0, 0, 0, None, 0, None) == 0


@pytest.mark.parametrize('N,T,null,ws,rc,msg', [
    (1, 1, False, None, -1, 'des_ga_order: N=1, need 2 <= N < 2^31'),
    (4, 0, False, None, -1, 'des_ga_order: T must be in [1, N = 4] (got 0)'),
    (4, 5, False, None, -1, 'des_ga_order: T must be in [1, N = 4] (got 5)'),
    (4, 2, True, None, -1, 'des_ga_order: NULL pointer'),
    (4, 2, False, 8, -4, None),
])
def test_ga_order_refuses(lib, N, T, null, ws, rc, msg):  # noqa: F811
    p = None if null else D
    assert lib.des_ga_order(p, p, N, T, D if ws else None, ws or 0, None) == rc
    need = lib.des_ga_order_workspace_bytes(N)
    assert _msg(lib) == (msg or 'des_ga_order: workspace 8 B < required %d B' % need)


def test_ga_order_workspace_covers_the_rank_path(lib):  # noqa: F811
    for N in (2, 2048, 2049, 65536):
        assert lib.des_ga_order_workspace_bytes(N) >= 3 * 4 * N + lib.des_rank_workspace_bytes(N, N)
    assert lib.des_ga_order_workspace_bytes(1) == 0


# ---- the wrappers ----------------------------------------------------------------------------------------------------
def test_wrappers_check_their_tensors():
    from distributedes_b200 import ops
    parents = torch.zeros((2, P))
    with pytest.raises(RuntimeError, match='parents must be a 2-D tensor'):
        ops.ga_rows(torch.zeros(P), 0, sigma=0.1, seed=0, generation=0, n_local=3)
    with pytest.raises(RuntimeError, match='parents must be torch.float32'):
        ops.ga_rows(parents.double(), 0, sigma=0.1, seed=0, generation=0, n_local=3)
    with pytest.raises(RuntimeError, match='members must be torch.int32'):
        ops.ga_rows(parents, 0, sigma=0.1, seed=0, generation=0, members=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(RuntimeError, match='out has %d entries, needs %d' % (2 * P, 3 * P)):
        ops.ga_rows(parents, 0, sigma=0.1, seed=0, generation=0, n_local=3, out=torch.zeros((2, P)))
    with pytest.raises(RuntimeError, match='give n_local or members'):
        ops.ga_rows(parents, 0, sigma=0.1, seed=0, generation=0)
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops.ga_rows(parents, 0, sigma=0.1, seed=0, generation=0, n_local=3)
    kw = dict(hidden=H, horizon=5, repetitions=2, sigma=0.1, clip=2.0, seed=1, n_local=3)
    with pytest.raises(RuntimeError, match='parents has %d entries, the \\(3,16,1\\) MLP needs n_parents x P = %d'
                                           % (2 * (P + 1), 2 * P)):
        ops.rollout_eval_ga(torch.zeros((2, P + 1)), 0, **kw)
    with pytest.raises(RuntimeError, match='episodes_out has 5 entries, needs 6'):
        ops.rollout_eval_ga(parents, 0, episodes_out=torch.zeros(5), **kw)
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops.rollout_eval_ga(parents, 0, **kw)
    with pytest.raises(RuntimeError, match='out must be torch.int32'):
        ops.ga_order(torch.zeros(4), 2, workspace=torch.zeros(1), out=torch.zeros(2))
    with pytest.raises(RuntimeError, match='fitness must be torch.float32'):
        ops.ga_order(torch.zeros(4, dtype=torch.float64), 2, workspace=torch.zeros(1))


# ---- the oracle ------------------------------------------------------------------------------------------------------
def _philox_scalar(c, k, rounds=7):
    """Philox4x32-R in Python integers, independent of nes_oracle's numpy loop."""
    c0, c1, c2, c3 = c
    k0, k1 = k
    for _ in range(rounds):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c3 ^ k1) & 0xFFFFFFFF, \
            p0 & 0xFFFFFFFF
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


@pytest.mark.parametrize('seed,gen', [(0, 0), (7, 3), ((5 << 32) + 11, 0xFFFFFFFF)])
def test_parent_draws_are_the_stream_5_words(seed, gen):
    members = [0, 1, 2, 5, 63, 1000, (1 << 28) - 1, (1 << 32) - 1]
    words = gao.parent_words(seed, gen, members)
    for m, x in zip(members, words):
        assert int(x) == _philox_scalar((0, m, gen, 5), (seed & 0xFFFFFFFF, seed >> 32))[0]
    for T, E in ((1, 0), (7, 2), (13, 13), (2048, 0)):
        p = gao.parents_of(seed, gen, members, T, E)
        for m, x, q in zip(members, words, p):
            assert q == (m if m < E else (int(x) * T) >> 32) and 0 <= q < T


def test_the_order_is_descending_with_ties_by_index_and_nan_last():
    f = np.array([1.0, np.nan, -0.0, 3.0, 0.0, 3.0, -np.inf, np.nan, 2.0], dtype=np.float32)
    assert gao.order(f, 9).tolist() == [3, 5, 8, 0, 2, 4, 6, 1, 7]
    assert gao.order(f, 2).tolist() == [3, 5]


def test_one_row_without_elites_is_the_nes_perturbation():
    theta = orc.synthetic_theta(3, H, 1, seed=2)
    rows = gao.member_rows(theta[None], 0, 0.05, 9, 4, np.arange(3, 8))
    np.testing.assert_array_equal(rows, orc.perturb(theta, np.float32(0.05), orc.noise(9, 4, 3, 5, P)))


# ---- genetic.train over the stand-in ---------------------------------------------------------------------------------
K = types.SimpleNamespace(**{k: v for m in (cpu_ops, cpu_ops_ga) for k, v in vars(m).items()
                             if not k.startswith('_') and callable(v)})


@pytest.fixture(autouse=True)
def _clear():
    cpu_ops_ga.CALLS.clear()


def _closed(N=6, T=3, E=1, gens=3, noise=0.0):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(H)
    c.pop_size, c.truncation, c.elites, c.max_generations, c.seed, c.sigma = N, T, E, gens, 5, 0.05
    c.repetitions = c.test_repetitions = 2
    c.action_noise_std = noise
    c.initial_weight = orc.synthetic_theta(3, H, 1, seed=1)
    return c


def _train(c, horizon=None, fused=True):
    from distributedes_b200 import genetic
    worker, ga = genetic.build(c, kernels=K, device='cpu', fused=fused)
    if horizon:
        worker.source.horizon = worker.source.T = horizon
    return genetic.train(c, worker, ga), ga


def _closed_chain(c, horizon):
    N, reps = c.pop_size, c.repetitions
    st = dict(stats=(np.zeros(3, np.float32), np.zeros(3, np.float32), np.float32(0)), totals=None)

    def evaluate(rows, g):
        ret, osum, osq, cnt = po.rollouts(rows, H, c.seed, g, np.arange(N), reps, st['stats'], horizon, c.clip,
                                          c.action_noise_std)
        st['totals'] = (osum, osq, cnt)
        return ret.mean(1).astype(np.float32), N * reps * horizon

    def test(theta, k):
        return np.mean(po.test_returns(theta, H, c.seed, k, c.test_repetitions, st['stats'], horizon, c.clip)
                       .astype(np.float32).astype(np.float64))

    def merge(g):
        st['stats'] = po.merge_totals(st['stats'], *st['totals'])
    return gao.train(c.initial_weight, sigma=c.sigma, N=N, T=c.truncation, E=c.elites, seed=c.seed,
                     generations=c.max_generations, evaluate=evaluate, test=test, merge=merge)


@pytest.mark.parametrize('fused', [True, False])
def test_closed_loop_train_equals_the_oracle_chain(fused):
    c = _closed(noise=0.1)
    (rewards, steps, _), ga = _train(c, horizon=6, fused=fused)
    chain = _closed_chain(c, 6)
    np.testing.assert_allclose(rewards, chain['rewards'], rtol=1e-6)
    assert steps == chain['steps']
    np.testing.assert_array_equal(ga.parents.numpy(), chain['tables'][-1])
    orders = [x['fitness'] for x in cpu_ops_ga.CALLS if x['op'] == 'ga_order']
    for f, want in zip(orders, chain['fitness']):
        np.testing.assert_array_equal(f.numpy(), want)
    ops = [x['op'] for x in cpu_ops_ga.CALLS]
    if fused:
        assert ops == ['rollout_eval_ga', 'ga_order', 'ga_rows'] * 3
        evals = [x for x in cpu_ops_ga.CALLS if x['op'] == 'rollout_eval_ga']
        assert [(x['n_parents'], x['n_elites'], x['generation'], x['member_offset']) for x in evals] == \
            [(1, 1, 0, 0), (3, 1, 1, 0), (3, 1, 2, 0)]
    else:
        assert ops == ['ga_rows', 'ga_order', 'ga_rows'] * 3


def test_tape_train_equals_the_oracle_chain():
    from distributedes_b200.config import PendulumConfig
    c = PendulumConfig(H, tape_len=8)
    c.pop_size, c.max_generations, c.seed, c.sigma = 11, 3, 2, 0.1
    (rewards, steps, _), ga = _train(c)
    assert (ga.T, ga.E) == (3, 2)                   # ceil(0.2 * 11) and the NEAT elitism
    env = c.env_fn()

    def fit(rows):
        return orc.tape_fitness(orc.forward(rows, env.obs, 3, H, 1), env.target, c.clip).astype(np.float32)
    chain = gao.train(c.initial_weight, sigma=c.sigma, N=11, T=3, E=2, seed=2, generations=3,
                      evaluate=lambda rows, g: (fit(rows), 11 * 8), test=lambda th, k: float(fit(th[None])[0]))
    np.testing.assert_allclose(rewards, chain['rewards'], rtol=1e-6)
    assert steps == chain['steps']
    np.testing.assert_array_equal(ga.parents.numpy(), chain['tables'][-1])


def test_host_stepped_train_equals_the_oracle_chain():
    from distributedes_b200.config import HostEnvConfig
    from distributedes_b200.envs import TEST_MEMBER, GymEnvBatch
    c = HostEnvConfig(SynthWalkEnv, hidden_size=H)
    c.pop_size, c.truncation, c.elites, c.max_generations, c.seed, c.sigma = 5, 2, 1, 2, 4, 0.1
    c.repetitions = c.test_repetitions = 2
    c.normalize_obs = False
    (rewards, steps, _), ga = _train(c)
    d0, A = c.state_dim, c.action_dim
    train_env, test_env = GymEnvBatch(SynthWalkEnv, 5 * 2, 4), GymEnvBatch(SynthWalkEnv, 2, 4)

    def evaluate(rows, g):
        ret, n, _ = po.episodes(rows, train_env, d0, H, A, c.clip, g, np.arange(5), 2, None, 4)
        return ret.mean(1).astype(np.float32), n

    def test(theta, k):
        ret, _, _ = po.episodes(theta[None], test_env, d0, H, A, c.clip, k, [TEST_MEMBER], 2, None, 4)
        return np.mean(ret[0])
    chain = gao.train(c.initial_weight, sigma=c.sigma, N=5, T=2, E=1, seed=4, generations=2, evaluate=evaluate,
                      test=test)
    np.testing.assert_allclose(rewards, chain['rewards'], rtol=1e-6)
    assert steps == chain['steps']
    np.testing.assert_array_equal(ga.parents.numpy(), chain['tables'][-1])


# ---- refusals --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('change,match', [
    (dict(mirrored=True), 'mirrored sampling'),
    (dict(pop_size=1), 'pop_size 1 < 2'),
    (dict(truncation=0), 'truncation 0 is not in \\[1, pop_size = 6\\]'),
    (dict(truncation=7), 'truncation 7 is not in \\[1, pop_size = 6\\]'),
    (dict(elites=4), 'elites 4 is not in \\[0, truncation = 3\\]'),
    (dict(elites=-1), 'elites -1 is not in \\[0, truncation = 3\\]'),
])
def test_refusals(change, match):
    from distributedes_b200 import genetic
    c = _closed()
    for k, v in change.items():
        setattr(c, k, v)
    for call in (lambda: genetic.train(c), lambda: genetic.Worker(c, device='cpu', kernels=K),
                 lambda: genetic.multi_runs(c, 1)):
        with pytest.raises(ValueError, match=match):
            call()
    if 'mirrored' not in change:
        with pytest.raises(ValueError, match=match):
            genetic.GeneticAlgorithm(c.initial_weight, 0.1, c.pop_size, c.truncation, c.elites, device='cpu', kernels=K)


def test_several_ranks_are_refused(monkeypatch):
    from distributedes_b200 import genetic
    monkeypatch.setattr(genetic.dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(genetic.dist, 'get_world_size', lambda *a: 2)
    with pytest.raises(ValueError, match='one process; the process group has world size 2'):
        genetic.GeneticAlgorithm(np.zeros(P), 0.1, 6, device='cpu', kernels=K)
    with pytest.raises(ValueError, match='world size 2'):
        genetic.train(_closed())


def test_defaults_follow_the_neat_reproduction_settings():
    from distributedes_b200 import genetic
    assert [genetic.selection_sizes(n) for n in (2, 5, 6, 30, 64, 1024)] == \
        [(2, 1, 1), (5, 1, 1), (6, 2, 2), (30, 6, 2), (64, 13, 2), (1024, 205, 2)]


def test_record_refuses_configs_that_are_not_closed_loop():
    from distributedes_b200 import genetic
    from distributedes_b200.config import PendulumConfig
    with pytest.raises(ValueError, match='closed-loop environments only'):
        genetic.record(PendulumConfig(H), np.zeros(P), None)
