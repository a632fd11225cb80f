"""Recorded closed-loop episodes without a GPU:

  - des_rollout_record[_solutions] refuse, before any CUDA work, every argument their evaluation counterparts refuse,
    with the counterpart's message under their own name, and trajectories past int64 elements;
  - n_local = 0 with NULL pointers does nothing;
  - the wrappers check each of the four trajectory outputs (dtype, element count, device) in ops._ptr;
  - the host logic of every surface over tests/cpu_ops_record.py: the seed, member offset and generation word each one
    launches with, and that what it records equals its test_returns / evaluate / run on the stand-in.
"""
import ctypes as C
import types

import numpy as np
import pytest

torch = pytest.importorskip('torch')

import cpu_ops
import cpu_ops_cma_sweep
import cpu_ops_record
import cpu_ops_sweep
from lib_fixture import lib  # noqa: F401
from oracle import nes_oracle as orc

D = C.c_void_p(256)          # never dereferenced: every case returns before any CUDA work


def _msg(lib):
    return lib.des_last_error().decode()


# ---- the entry points ------------------------------------------------------------------------------------------------
# case -> (env, H, repetitions, tape_len, member_offset, n_local, noiseless, mirrored, null pointers, totals, workspace)
CASES = {
    'bad_env': (1, 32, 10, 200, 0, 2, 0, 0, False, False, 0),
    'bad_width': (0, 48, 10, 200, 0, 2, 0, 0, False, False, 0),
    'reps_0': (0, 32, 0, 200, 0, 2, 0, 0, False, False, 0),
    'reps_11': (0, 32, 11, 200, 0, 2, 0, 0, False, False, 0),
    'tape_0': (0, 32, 10, 0, 0, 2, 0, 0, False, False, 0),
    'neg_offset': (0, 32, 10, 200, -2, 2, 0, 0, False, False, 0),
    'past_2^28': (0, 32, 10, 200, (1 << 28) - 2, 4, 0, 0, False, False, 0),
    'odd_pairs': (0, 32, 10, 200, 1, 2, 0, 1, False, False, 0),
    'mirrored_noiseless': (0, 32, 10, 200, 0, 2, 1, 1, False, False, 0),
    'null_count': (0, 32, 10, 200, 0, 2, 0, 0, True, False, 0),
    'small_workspace': (0, 32, 10, 200, 0, 2, 0, 0, False, True, 8),
    'null_zero_count': (0, 32, 10, 200, 0, 0, 0, 0, True, False, 0),
}


def _dims(_lib, H, T):
    return _lib.Dims(3, H, 1, T)


def _pair(lib, kind, case, traj=(None, None, None, None)):
    """(counterpart status and message, recording status and message) for one case."""
    from distributedes_b200 import _lib
    env, H, reps, T, off, n, noiseless, mirrored, null, totals, ws = CASES[case]
    p = None if null else D
    tot = D if totals else None
    if kind == 'theta':
        ev = lib.des_rollout_eval_mirrored if mirrored else lib.des_rollout_eval
        rc = ev(p, None, tot, p, None, env, _dims(_lib, H, T), reps, 0.1, 2.0, 0.0, 0, 0, None, off, n, noiseless,
                D if ws else None, ws, None)
        a = (rc, _msg(lib) if rc else None)
        rc = lib.des_rollout_record(p, None, tot, p, None, env, _dims(_lib, H, T), reps, 0.1, 2.0, 0.0, 0, 0, None, off, n,
                                    noiseless, mirrored, *traj, D if ws else None, ws, None)
    else:
        rc = lib.des_rollout_eval_solutions(p, None, tot, p, None, env, _dims(_lib, H, T), reps, 2.0, 0.0, 0, 0, off, n,
                                            D if ws else None, ws, None)
        a = (rc, _msg(lib) if rc else None)
        rc = lib.des_rollout_record_solutions(p, None, tot, p, None, env, _dims(_lib, H, T), reps, 2.0, 0.0, 0, 0, off, n,
                                              *traj, D if ws else None, ws, None)
    return a, (rc, _msg(lib) if rc else None)


@pytest.mark.parametrize('case', list(CASES))
@pytest.mark.parametrize('kind', ['theta', 'rows'])
@pytest.mark.parametrize('traj', ['null', 'all'])
def test_recordings_refuse_what_their_evaluations_refuse(lib, kind, case, traj):  # noqa: F811
    if kind == 'rows' and CASES[case][7]:
        pytest.skip('explicit rows have no mirrored pairs')
    ev, rec = _pair(lib, kind, case, (None,) * 4 if traj == 'null' else (D,) * 4)
    assert ev[0] != 0 or case == 'null_zero_count', (case, ev)
    assert rec[0] == ev[0], (case, ev, rec)
    if ev[1] is not None:
        name = 'des_rollout_record' if kind == 'theta' else 'des_rollout_record_solutions'
        assert rec[1] == ev[1].replace(ev[1].split(':')[0], name, 1), (ev, rec)


@pytest.mark.parametrize('kind', ['theta', 'rows'])
@pytest.mark.parametrize('which', [0, 1], ids=['states', 'obs'])
def test_oversized_trajectories_are_refused(lib, kind, which):  # noqa: F811
    """(2^28 - 16) members x 10 episodes x (2^31 - 1) steps x width 2 or 3 is past 2^63 elements.  Width 1 (actions,
    rewards) stays below 2^63 at every size the member range allows, so it is never refused."""
    from distributedes_b200 import _lib
    traj = [None] * 4
    traj[which] = D
    n, T = (1 << 28) - 16, (1 << 31) - 1
    dims = _lib.Dims(3, 32, 1, T)
    if kind == 'theta':
        rc = lib.des_rollout_record(D, None, None, D, None, 0, dims, 10, 0.1, 2.0, 0.0, 0, 0, None, 0, n, 0, 0, *traj,
                                    None, 0, None)
        name = 'des_rollout_record'
    else:
        rc = lib.des_rollout_record_solutions(D, None, None, D, None, 0, dims, 10, 2.0, 0.0, 0, 0, 0, n, *traj, None, 0,
                                              None)
        name = 'des_rollout_record_solutions'
    assert rc == -1
    assert _msg(lib) == ('%s: trajectories of %d members x 10 episodes x %d steps exceed int64 elements' % (name, n, T))


# ---- the wrappers ----------------------------------------------------------------------------------------------------
TRAJ = {'states_out': (torch.float64, 2), 'obs_out': (torch.float32, 3), 'actions_out': (torch.float32, 1),
        'rewards_out': (torch.float64, 1)}


def _wrapper_call(kind, **traj):
    from distributedes_b200 import ops
    n, reps, T = 2, 3, 5
    kw = dict(hidden=16, horizon=T, repetitions=reps, clip=2.0, seed=1, out=torch.empty(n))
    if kind == 'theta':
        return ops.rollout_record(torch.zeros(orc.param_count(3, 16, 1)), sigma=0.1, n_local=n, **kw, **traj)
    return ops.rollout_record_solutions(torch.zeros((n, orc.param_count(3, 16, 1))), **kw, **traj)


@pytest.mark.parametrize('kind', ['theta', 'rows'])
@pytest.mark.parametrize('name', list(TRAJ))
def test_wrappers_check_every_trajectory(kind, name):
    dtype, width = TRAJ[name]
    good = 2 * 3 * 5 * width
    wrong = torch.float32 if dtype == torch.float64 else torch.float64
    with pytest.raises(RuntimeError, match='%s must be %s' % (name, dtype)):
        _wrapper_call(kind, **{name: torch.empty(good, dtype=wrong)})
    with pytest.raises(RuntimeError, match='%s has %d entries, needs %d' % (name, good + 1, good)):
        _wrapper_call(kind, **{name: torch.empty(good + 1, dtype=dtype)})
    with pytest.raises(RuntimeError, match='%s is on meta, the op runs on cpu' % name):
        _wrapper_call(kind, **{name: torch.empty(good, dtype=dtype, device='meta')})
    with pytest.raises(RuntimeError, match='CPU tensor'):          # every check passed: only the device is left
        _wrapper_call(kind, **{name: torch.empty(good, dtype=dtype)})


# ---- host logic over the stand-in ------------------------------------------------------------------------------------
def _kernels(*mods):
    ns = {}
    for m in mods + (cpu_ops_record,):
        ns.update({k: v for k, v in vars(m).items() if not k.startswith('_') and callable(v)})
    return types.SimpleNamespace(**ns)


K = _kernels(cpu_ops)
K_SWEEP = _kernels(cpu_ops_sweep)
K_CMA_SWEEP = _kernels(cpu_ops_cma_sweep)
H, T = 16, 6


def _theta():
    return orc.synthetic_theta(3, H, 1, seed=3)


@pytest.fixture(autouse=True)
def _calls():
    cpu_ops_record.CALLS.clear()
    yield


def _engine(mirrored=False, noise=0.0):
    from distributedes_b200.engine import RolloutEngine
    eng = RolloutEngine(hidden=H, pop_size=6, theta0=_theta(), sigma=0.1, learning_rate=0.05, repetitions=3, horizon=T,
                        action_noise_std=noise, seed=11, mirrored=mirrored, kernels=K, device='cpu')
    eng.generation()
    eng.generation()
    return eng


@pytest.mark.parametrize('mirrored', [False, True])
def test_rollout_engine_records_with_its_keys_and_advances_nothing(mirrored):
    eng = _engine(mirrored)
    state = eng.state.clone()
    tr = eng.record_test_episodes()
    (c,) = cpu_ops_record.CALLS
    assert (c['noiseless'], c['mirrored'], c['member_offset'], c['n_local'], c['generation'], c['seed']) == \
        (True, False, 0, 1, 2, 11)
    assert torch.equal(c['obs_stats'], eng.obs_stats)
    assert tr.states.shape == (3, T, 2) and tr.obs.shape == (3, T, 3) and tr.actions.shape == (3, T, 1)
    assert np.array_equal(tr.returns.astype(np.float64), eng.test_returns())
    rec = eng.record_members(2, 4)
    c = cpu_ops_record.CALLS[-1]
    assert (c['noiseless'], c['mirrored'], c['member_offset'], c['n_local'], c['generation']) == \
        (False, mirrored, 2, 4, 2)
    assert torch.equal(eng.state, state)
    totals = eng.obs_totals.clone()
    fit = eng.evaluate().numpy()
    assert rec.returns.shape == (4, 3)
    assert np.array_equal(rec.returns.astype(np.float64).mean(1).astype(np.float32), fit[2:6]) or \
        np.allclose(rec.returns.mean(1), fit[2:6], rtol=1e-6)
    assert not torch.equal(totals, torch.zeros_like(totals))
    with pytest.raises(ValueError, match='not in the population'):
        eng.record_members(4, 3)


def test_a_tape_engine_is_refused():
    from distributedes_b200.engine import NESEngine
    eng = NESEngine(state_dim=3, hidden=H, action_dim=1, pop_size=4, theta0=_theta(), obs=np.zeros((5, 3)),
                    target=np.zeros((5, 1)), sigma=0.1, learning_rate=0.1, kernels=K, device='cpu')
    with pytest.raises(TypeError, match='closed-loop environments only'):
        eng.record_test_episodes()


@pytest.mark.parametrize('sweep', [False, True])
def test_runs_engine_keys_each_run(sweep):
    from distributedes_b200.engine import RolloutRunsEngine
    kw = dict(seeds=[5, 9, 13], sigma=[0.1, 0.05, 0.2], action_noise_std=[0.2, 0.0, 0.3]) if sweep else \
        dict(seed=7, sigma=0.1, action_noise_std=0.2)
    eng = RolloutRunsEngine(hidden=H, pop_size=4, runs=3, theta0=_theta(), learning_rate=0.05, repetitions=3, horizon=T,
                            kernels=K_SWEEP, device='cpu', **kw)
    eng.generation()
    for r in range(3):
        eng.record_test_episodes(r)
        c = cpu_ops_record.CALLS[-1]
        want = (([5, 9, 13][r], [0.2, 0.0, 0.3][r], 0) if sweep else (7, 0.2, r))
        assert (c['seed'], c['action_noise_std'], c['member_offset']) == want
        assert (c['noiseless'], c['generation'], c['n_local']) == (True, 1, 1)
        assert torch.equal(c['theta'], eng.theta[r]) and torch.equal(c['obs_stats'], eng.obs_stats[r])
    with pytest.raises(ValueError, match='not in'):
        eng.record_test_episodes(3)


def test_runs_engine_records_equal_test_returns_without_action_noise():
    from distributedes_b200.engine import RolloutRunsEngine
    eng = RolloutRunsEngine(hidden=H, pop_size=4, runs=2, theta0=_theta(), learning_rate=0.05, repetitions=3, horizon=T,
                            seeds=[5, 9], sigma=0.1, kernels=K_SWEEP, device='cpu')
    eng.generation()
    ret = eng.test_returns()
    for r in range(2):
        assert np.array_equal(eng.record_test_episodes(r).returns.astype(np.float64), ret[r])


def _cma_config(seed=3, noise=0.0):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(H)
    c.seed, c.action_noise_std, c.pop_size, c.repetitions, c.test_repetitions = seed, noise, 4, 2, 3
    c.initial_weight = _theta()
    c.tape_len = T
    return c


def test_cma_worker_keys_the_next_test_and_advances_nothing():
    from distributedes_b200 import cma_es
    from distributedes_b200.utils import StaticNormalizer
    c = _cma_config()
    w = cma_es.Worker(0, StaticNormalizer(3), None, None, None, c, device='cpu', kernels=K)
    w.source.horizon = T
    w.test_returns(torch.from_numpy(_theta()), 3)
    tr = w.record_test_episodes(_theta(), 3)
    c0 = cpu_ops_record.CALLS[-1]
    assert (c0['generation'], c0['noiseless'], c0['member_offset'], w.tests_run) == (1, True, 0, 1)
    assert np.array_equal(tr.returns.astype(np.float64), w.test_returns(torch.from_numpy(_theta()), 3))
    rows = torch.from_numpy(np.tile(_theta(), (3, 1)))
    rec = w.record_solutions(rows, member_offset=5, generation=2)
    c1 = cpu_ops_record.CALLS[-1]
    assert (c1['op'], c1['member_offset'], c1['generation'], c1['n_local']) == ('rollout_record_solutions', 5, 2, 3)
    assert np.allclose(-rec.returns.mean(1), w.run(rows, 5, 2).numpy(), rtol=1e-6)


def test_cma_sweep_worker_keys_each_run_at_offset_0():
    from distributedes_b200 import cma_es
    configs = [_cma_config(3, 0.2), _cma_config(8, 0.0)]
    w = cma_es.SweepWorker(configs, device='cpu', kernels=K_CMA_SWEEP)
    w.tests_run = 4
    for r in range(2):
        w.record_test_episodes(_theta(), r)
        c = cpu_ops_record.CALLS[-1]
        assert (c['seed'], c['action_noise_std'], c['member_offset'], c['generation'], c['noiseless']) == \
            ([3, 8][r], [0.2, 0.0][r], 0, 4, True)
    assert w.tests_run == 4


def test_trainer_records_refuse_other_configs():
    from distributedes_b200 import cma_es, natural_es
    from distributedes_b200.config import SynthTapeConfig
    c = SynthTapeConfig(16) if callable(SynthTapeConfig) else None
    for fn in (natural_es.record, cma_es.record):
        with pytest.raises(ValueError, match='closed-loop environments only'):
            fn(c, None, None)
