"""Recorded closed-loop episodes (des_rollout_record[_solutions], the RecordArgs instantiations of rollout_pendulum_kernel)
on the GPU:

  1. the outputs shared with the evaluation are bit-equal to des_rollout_eval, _mirrored and _solutions;
  2. the return and totals identities of include/des_b200.h hold bit for bit, with any subset of trajectories NULL;
  3. the trajectories against the oracle: the reset states exactly, each observation to 1 fp32 ulp of gym's observation of
     the recorded state, each step to a few fp64 ulp of gym's dynamics (the device sincos), each action within
     KAPPA[H] * closed_loop_bound of the fp64 forward (test_gpu_rollout_actions.py's bounds, without its recovery
     resolution) and within the clip, NaN kept;
  4. the torques oracle/rollout_probe.py recovers from the totals equal the recorded actions clamped to +-2;
  5. every surface records what its test_returns / evaluate / run computes, and train() on the closed-loop golden config
     reproduces its rewards from recordings made at each test point.
"""
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import forward_error as fe
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from oracle import rollout_probe as rp

pytestmark = pytest.mark.gpu

SEED, GEN, SIGMA = 2026, 4, 0.1
KAPPA = {16: 1.7, 32: 0.5, 64: 0.15, 96: 0.045, 128: 0.028}          # test_gpu_rollout_actions.py
STATS = (np.float32([-0.2, 0.01, 0.3]), np.float32([0.5, 0.4, 20.0]), np.float32(32000))
TOP = (1 << 28) - 1
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def ops():
    from distributedes_b200 import ops as _ops
    return _ops


def dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).cuda()


def _stats_tensor(stats):
    return None if stats is None else dev(np.concatenate([stats[0], stats[1], [stats[2]]]))


def _theta(H):
    return orc.synthetic_theta(3, H, 1, seed=H)


def _rows(H, n, seed):
    rs = np.random.RandomState(seed)
    return (_theta(H)[None, :] + 0.3 * rs.randn(n, orc.param_count(3, H, 1))).astype(np.float32)


def launch(mode, H, reps, horizon, n, offset=0, stats=None, noise=0.0, clip=2.0, rows=None, traj=(1, 1, 1, 1)):
    """The evaluation of `mode` and its recording on the same arguments.  Returns (evaluation outputs, recording outputs,
    trajectories as numpy arrays or None where the pointer was NULL, the weight rows the members used)."""
    o, f32, f64 = ops(), torch.float32, torch.float64
    st = _stats_tensor(stats)
    kw = dict(hidden=H, horizon=horizon, repetitions=reps, clip=clip, action_noise_std=noise, seed=SEED, generation=GEN,
              obs_stats=st)

    def outs():
        return dict(out=torch.full((n,), 7.0, dtype=f32, device='cuda'),
                    episodes_out=torch.full((n, reps), 7.0, dtype=f32, device='cuda'),
                    totals_out=torch.full((7,), 7.0, dtype=f64, device='cuda'))
    tr = dict(states_out=torch.full((n, reps, horizon, 2), np.nan, dtype=f64, device='cuda'),
              obs_out=torch.full((n, reps, horizon, 3), np.nan, dtype=f32, device='cuda'),
              actions_out=torch.full((n, reps, horizon, 1), np.nan, dtype=f32, device='cuda'),
              rewards_out=torch.full((n, reps, horizon), np.nan, dtype=f64, device='cuda'))
    tr = {k: (v if on else None) for (k, v), on in zip(tr.items(), traj)}
    e, r = outs(), outs()
    if mode == 'rows':
        sol = dev(rows if rows is not None else _rows(H, n, offset % 1000 + H))
        o.rollout_eval_solutions(sol, member_offset=offset, **kw, **e)
        o.rollout_record_solutions(sol, member_offset=offset, **kw, **r, **tr)
        flat = sol.cpu().numpy()
    else:
        theta = dev(_theta(H))
        noiseless = mode == 'test'
        nk = dict(sigma=0.0 if noiseless else SIGMA, member_offset=offset, n_local=n, noiseless=noiseless)
        (o.rollout_eval_mirrored if mode == 'mirrored' else o.rollout_eval)(theta, **nk, **kw, **e)
        o.rollout_record(theta, mirrored=mode == 'mirrored', **nk, **kw, **r, **tr)
        if noiseless:
            flat = np.tile(_theta(H), (n, 1))
        elif mode == 'mirrored':
            flat = o.nes_perturb_mirrored(theta, n, SIGMA, SEED, GEN, member_offset=offset).cpu().numpy()
        else:
            flat = o.nes_perturb(theta, n, SIGMA, SEED, GEN, member_offset=offset).cpu().numpy()
    np_ = lambda d: {k: (None if v is None else v.cpu().numpy()) for k, v in d.items()}      # noqa: E731
    return np_(e), np_(r), np_(tr), flat


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


# ---- 1. the evaluation's outputs, bit for bit ------------------------------------------------------------------------
# id: (mode, H, repetitions, horizon, n_local, member_offset, stats, action noise)
SHARED = {
    'nes-h16-r10-t200': ('nes', 16, 10, 200, 5, 3, None, 0.0),
    'nes-h32-r3-t200-stats-noise': ('nes', 32, 3, 200, 4, 11, STATS, 0.3),
    'nes-h64-r1-t1': ('nes', 64, 1, 1, 6, 0, STATS, 0.0),
    'nes-h96-r10-t200-noise': ('nes', 96, 10, 200, 3, 40, None, 0.3),
    'nes-h128-r3-t200-stats': ('nes', 128, 3, 200, 3, 7, STATS, 0.0),
    'mirrored-h32-r10-t200-stats-noise': ('mirrored', 32, 10, 200, 6, 8, STATS, 0.3),
    'mirrored-h128-r1-t1': ('mirrored', 128, 1, 1, 4, 2, None, 0.0),
    'rows-h16-r3-t1-noise': ('rows', 16, 3, 1, 5, 9, None, 0.3),
    'rows-h64-r10-t200-stats-noise': ('rows', 64, 10, 200, 4, 21, STATS, 0.3),
    'rows-h96-r1-t200': ('rows', 96, 1, 200, 3, 0, None, 0.0),
    'test-h64-r10-t200-stats-noise': ('test', 64, 10, 200, 1, 0, STATS, 0.3),
    'test-h128-r3-t200-offset': ('test', 128, 3, 200, 1, 5, None, 0.3),
    'top-member-h32-r10': ('nes', 32, 10, 200, 1, TOP, None, 0.3),
    'top-member-rows-h64-r3': ('rows', 64, 3, 200, 2, TOP - 1, STATS, 0.3),
    'pop-2048-h32-r10': ('nes', 32, 10, 200, 2048, 0, STATS, 0.3),
}


@pytest.mark.parametrize('name', list(SHARED))
def test_recording_writes_the_evaluations_outputs_bit_for_bit(name):
    mode, H, reps, T, n, off, stats, noise = SHARED[name]
    e, r, _, _ = launch(mode, H, reps, T, n, off, stats, noise)
    for k in ('out', 'episodes_out', 'totals_out'):
        assert np.array_equal(_bits(e[k]), _bits(r[k])), (name, k)


def test_a_nan_weight_row_records_nan_and_matches_the_evaluation():
    rows = _rows(32, 3, 5)
    rows[1, 40] = np.nan
    e, r, tr, _ = launch('rows', 32, 3, 200, 3, 0, None, 0.0, rows=rows)
    for k in ('out', 'episodes_out', 'totals_out'):
        assert np.array_equal(_bits(e[k]), _bits(r[k])), k
    assert np.isnan(tr['actions_out'][1]).all() and np.isnan(r['episodes_out'][1]).all()
    assert not np.isnan(tr['actions_out'][[0, 2]]).any()
    assert np.isnan(tr['rewards_out'][1]).all()


# ---- 2. the identities -----------------------------------------------------------------------------------------------
def _fp64_returns(rewards):
    """fp64 sums over t in order from 0.0, [n, reps]."""
    tot = np.zeros(rewards.shape[:2])
    for t in range(rewards.shape[2]):
        tot = tot + rewards[:, :, t]
    return tot


def _totals(obs):
    """The documented order: per member, episodes in order of (steps in order), members in order."""
    n, reps, T, d0 = obs.shape
    o = obs.astype(np.float64)
    out = np.zeros(2 * d0 + 1)
    for i in range(n):
        mem = np.zeros(2 * d0)
        for e in range(reps):
            s, q = np.zeros(d0), np.zeros(d0)
            for t in range(T):
                s = s + o[i, e, t]
                q = q + o[i, e, t] * o[i, e, t]
            mem = mem + np.concatenate([s, q])
        out[:2 * d0] = out[:2 * d0] + mem
        out[2 * d0] += float(reps * T)
    return out


@pytest.mark.parametrize('traj', [(1, 1, 1, 1), (0, 1, 0, 1), (1, 0, 1, 0), (0, 0, 0, 1), (0, 0, 0, 0)],
                         ids=['all', 'obs-rewards', 'states-actions', 'rewards', 'none'])
@pytest.mark.parametrize('mode', ['nes', 'rows', 'test'])
def test_return_and_totals_identities(mode, traj):
    n = 1 if mode == 'test' else 3
    e, r, tr, _ = launch(mode, 32, 10, 200, n, 4, STATS, 0.3, traj=traj)
    for k in ('out', 'episodes_out', 'totals_out'):
        assert np.array_equal(_bits(e[k]), _bits(r[k])), k
    if tr['rewards_out'] is not None:
        ret = _fp64_returns(tr['rewards_out'])
        assert np.array_equal(_bits(ret.astype(np.float32)), _bits(r['episodes_out']))
        if mode != 'test':
            fit = np.zeros(n)
            for ep in range(10):
                fit = fit + ret[:, ep]
            assert np.array_equal(_bits((fit / 10).astype(np.float32)), _bits(r['out']))
    if tr['obs_out'] is not None:
        assert np.array_equal(_bits(_totals(tr['obs_out'])), _bits(r['totals_out']))


# ---- 3. against the oracle -------------------------------------------------------------------------------------------
ORACLE = {
    'nes-h16': ('nes', 16, 10, 3, None, 0.0, 2.0),
    'nes-h64-stats-noise': ('nes', 64, 10, 6, STATS, 0.3, 2.0),
    'mirrored-h32-noise': ('mirrored', 32, 10, 7, None, 0.3, 2.0),
    'rows-h128-stats': ('rows', 128, 10, 40, STATS, 0.0, 2.0),
    'rows-h96-clip-0.5': ('rows', 96, 3, 41, None, 0.3, 0.5),
    'test-h32-noise': ('test', 32, 10, 2, None, 0.3, 2.0),
    'top-member-h64': ('nes', 64, 10, TOP, None, 0.3, 2.0),
}


def _ulp64(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)))


@pytest.mark.parametrize('name', list(ORACLE))
def test_trajectories_against_the_oracle(name):
    mode, H, reps, member, stats, noise, clip = ORACLE[name]
    n = 2 if mode == 'mirrored' else 1
    off = member - 1 if mode == 'mirrored' else member
    e, r, tr, flat = launch(mode, H, reps, 200, n, off, stats, noise, clip)
    i = n - 1                                                   # the member checked (a mirrored pair's odd one)
    states, obs = tr['states_out'][i], tr['obs_out'][i]
    act, rew = tr['actions_out'][i, ..., 0], tr['rewards_out'][i]
    # resets, exactly
    th0, td0 = po.reset_states(SEED, GEN, [po.TEST_MEMBER if mode == 'test' else off + i], reps)
    assert np.array_equal(states[:, 0, 0], th0[0]) and np.array_equal(states[:, 0, 1], td0[0])
    # observations: gym's of the recorded state, to 1 fp32 ulp
    ref = po.pendulum_obs(states[..., 0], states[..., 1]).astype(np.float32)
    assert np.all(np.abs(obs.astype(np.float64) - ref) <= np.spacing(np.abs(ref)).astype(np.float64)), name
    # dynamics: a few fp64 ulp (the device sincos; the fp64 modulo of th + pi)
    nth, nthd, rw = po.pendulum_step(states[:, :-1, 0], states[:, :-1, 1], act[:, :-1].astype(np.float64))
    assert np.all(np.abs(nth - states[:, 1:, 0]) <= 8 * _ulp64(np.abs(nth) + 1.0)), name
    assert np.all(np.abs(nthd - states[:, 1:, 1]) <= 8 * _ulp64(np.abs(nthd) + 1.0)), name
    tol_r = 64 * _ulp64(np.abs(states[:, :-1, 0]) + np.pi) * (2 * np.pi + 1) + 8 * _ulp64(rw)
    assert np.all(np.abs(rw - rew[:, :-1]) <= tol_r), name
    # actions: within the clip, and within KAPPA * B of the fp64 forward of the member's weights at the recorded obs
    assert np.all(np.abs(act) <= np.float32(clip))
    noise_member = off + i
    z0, z1 = rp.action_normals(SEED, GEN, noise_member, 200)
    std32 = float(np.float32(noise))
    nz, nerr = std32 * z0[:reps], std32 * rp.normal_error(z0[:reps], z1[:reps])
    x = obs.astype(np.float64)
    a_star = fe.closed_loop_actions(flat[i], x, 3, H, 1, stats, nz[..., None])[..., 0]
    B = fe.closed_loop_bound(flat[i], x, 3, H, 1, stats, nz[..., None], nerr[..., None])[..., 0]
    ref_a = np.clip(a_star, -clip, clip)
    d = np.abs(act.astype(np.float64) - ref_a)
    half = np.spacing(np.abs(act)).astype(np.float64) / 2                  # the action's own fp32 rounding
    assert np.all(d <= KAPPA[H] * B + half), (name, float(np.max(d / (KAPPA[H] * B + half))))


# ---- 4. two routes to the same torques -------------------------------------------------------------------------------
def test_probe_recovers_the_recorded_torques():
    """oracle/rollout_probe.py's torques from double differences of the totals, at every step 0..39 of member 3's ten
    episodes, against the recorded actions clamped to +-2: equal within the probe's resolution."""
    from test_gpu_rollout_actions import Probe
    p = Probe('nes', 32, range(0, 41), None, 0.0, 2.0, 3)
    _, _, tr, _ = launch('nes', 32, 10, 200, 1, 3, None, 0.0)
    act = tr['actions_out'][0, :, :40, 0].astype(np.float64)
    u, res, valid = (x[:, :40] for x in rp.torques(p.obs, p.err))
    assert valid.sum() > 300
    assert np.all(np.where(valid, np.abs(u - np.clip(act, -2.0, 2.0)), 0.0) <= res)


# ---- 5. the surfaces -------------------------------------------------------------------------------------------------
def _fitness_of(traj):
    ret = _fp64_returns(traj.rewards)
    s = np.zeros(ret.shape[0])
    for ep in range(ret.shape[1]):
        s = s + ret[:, ep]
    return (s / ret.shape[1]).astype(np.float32)


def _trained_engine(mirrored):
    from distributedes_b200.engine import RolloutEngine
    eng = RolloutEngine(hidden=32, pop_size=16, theta0=_theta(32), sigma=SIGMA, learning_rate=0.05, repetitions=4,
                        action_noise_std=0.2, seed=SEED, mirrored=mirrored, use_graph=False)
    eng.generation()                                     # statistics and a generation word other than 0
    return eng


@pytest.mark.parametrize('mirrored', [False, True], ids=['plain', 'mirrored'])
def test_rollout_engine_surfaces(mirrored):
    from distributedes_b200 import ops as o
    eng = _trained_engine(mirrored)
    word = o.read_state(eng.state)['generation']
    tr = eng.record_test_episodes()
    assert np.array_equal(tr.returns.astype(np.float64), eng.test_returns())
    assert tr.states.shape == (4, 200, 2)
    rec = eng.record_members(4, 8)
    assert o.read_state(eng.state)['generation'] == word
    fit = eng.evaluate().cpu().numpy()
    assert np.array_equal(_bits(_fitness_of(rec)), _bits(fit[4:12]))


@pytest.mark.parametrize('sweep', [False, True], ids=['batch', 'sweep'])
def test_rollout_runs_engine_records_every_runs_test_episodes(sweep):
    from distributedes_b200.engine import RolloutRunsEngine
    kw = dict(seeds=[5, 9, 13], sigma=[0.1, 0.05, 0.2], action_noise_std=[0.2, 0.0, 0.3]) if sweep else \
        dict(seed=SEED, sigma=SIGMA, action_noise_std=0.2)
    eng = RolloutRunsEngine(hidden=32, pop_size=8, runs=3, theta0=_theta(32), learning_rate=0.05, repetitions=4,
                            use_graph=False, **kw)
    eng.generation()
    ret = eng.test_returns()
    for r in range(3):
        assert np.array_equal(eng.record_test_episodes(r).returns.astype(np.float64), ret[r]), r


def _cma_config(seed=3, noise=0.2):
    from distributedes_b200.config import ClosedLoopPendulumConfig
    c = ClosedLoopPendulumConfig(32)
    c.seed, c.action_noise_std, c.pop_size, c.repetitions, c.test_repetitions = seed, noise, 8, 3, 5
    c.initial_weight = _theta(32)
    return c


def test_cma_worker_surfaces():
    from distributedes_b200 import cma_es
    from distributedes_b200.utils import StaticNormalizer
    c = _cma_config()
    w = cma_es.Worker(0, StaticNormalizer(3), None, None, None, c)
    w.obs_stats.copy_(_stats_tensor(STATS))
    w.test_returns(dev(_theta(32)).reshape(1, -1), 5)                # tests_run = 1
    sol = _rows(32, 1, 3)[0]
    tr = w.record_test_episodes(sol)
    assert w.tests_run == 1
    assert np.array_equal(tr.returns.astype(np.float64), w.test_returns(dev(sol).reshape(1, -1), 5))
    rows = dev(_rows(32, 6, 8))
    rec = w.record_solutions(rows, member_offset=2, generation=7)
    cost = w.run(rows, member_offset=2, generation=7).cpu().numpy()
    assert np.array_equal(_bits(-_fitness_of(rec)), _bits(cost))


def test_cma_sweep_worker_records_every_runs_test_episodes():
    from distributedes_b200 import cma_es
    configs = [_cma_config(3, 0.2), _cma_config(8, 0.0), _cma_config(11, 0.4)]
    w = cma_es.SweepWorker(configs)
    w.obs_stats.copy_(_stats_tensor(STATS).repeat(3, 1) * torch.tensor([[1.0], [0.5], [2.0]], device='cuda'))
    sols = dev(_rows(32, 3, 4))
    w.test_returns(sols, 5, np.ones(3, dtype=bool))
    recs = [w.record_test_episodes(sols[r], r) for r in range(3)]
    ret = w.test_returns(sols, 5, np.ones(3, dtype=bool))
    for r in range(3):
        assert np.array_equal(recs[r].returns.astype(np.float64), ret[r]), r


def test_train_rewards_from_recordings_on_the_closed_loop_golden():
    """natural_es.train on train_closed_pend.npz's config: at every test point, natural_es.record on the engine records
    the episodes whose mean train() logs."""
    from distributedes_b200 import natural_es
    from test_gpu_goldens import device_rollouts
    g = dict(np.load(os.path.join(GOLDEN, 'train_closed_pend.npz')))
    cfg = device_rollouts(g)
    eng = natural_es.build_engine(cfg)
    means, real = [], eng.test_returns

    def spy(solution=None, repetitions=None):
        means.append(np.mean(natural_es.record(cfg, solution, None, engine=eng).returns.astype(np.float64)))
        return real(solution, repetitions)
    eng.test_returns = spy
    rewards, _, _ = natural_es.train(cfg, engine=eng)
    assert len(means) == len(rewards) and [float(m) for m in means] == [float(x) for x in rewards]
    first = natural_es.record(cfg, None, None)               # no engine: keyed as train()'s first test()
    assert float(np.mean(first.returns.astype(np.float64))) == float(rewards[0])


def test_cma_record_keys_as_the_first_test_of_train():
    from distributedes_b200 import cma_es
    c = _cma_config()
    tr = cma_es.record(c, c.initial_weight, None)
    mean, _ = cma_es.test(c, c.initial_weight, None)
    assert float(np.mean(tr.returns.astype(np.float64))) == float(mean)
