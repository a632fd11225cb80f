"""Oracle-backed stand-in for the two recording ops (ops.rollout_record, ops.rollout_record_solutions), on CPU tensors.
TEST-ONLY: the episodes of rollout_pendulum_kernel restated with oracle/pendulum_oracle.py's reset_states,
pendulum_obs, pendulum_step, policy_actions and action_noise, step by step, writing the trajectories the library
documents.  Episode (i, e) resets as member member_offset + i (test episodes: TEST_MEMBER) and draws its action noise
as member member_offset + i.  The fitness, returns and totals are those of cpu_ops' evaluation stand-ins on the same
arguments (their fp64 return sums in step order, their mean over the repetitions), so a surface recorded through this
module can be compared with the same surface evaluated through cpu_ops.  Every call is appended to CALLS."""
import numpy as np
import torch

from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

CALLS = []


def _episodes(rows, H, seed, gen, reset_members, noise_offset, reps, horizon, clip, act_noise, stats):
    n = rows.shape[0]
    th, thd = po.reset_states(seed, gen, reset_members, reps)
    states = np.zeros((n, reps, horizon, 2))
    obs = np.zeros((n, reps, horizon, 3), dtype=np.float32)
    act = np.zeros((n, reps, horizon, 1), dtype=np.float32)
    rew = np.zeros((n, reps, horizon))
    ret = np.zeros((n, reps))
    for t in range(horizon):
        states[:, :, t, 0], states[:, :, t, 1] = th, thd
        o = po.pendulum_obs(th, thd).astype(np.float32)
        obs[:, :, t] = o
        a = po.policy_actions(rows, o, np.ones((n, reps), dtype=bool), 3, H, 1, clip, stats, act_noise, seed, gen,
                              noise_offset, t)
        act[:, :, t] = a.astype(np.float32)
        th, thd, r = po.pendulum_step(th, thd, a[..., 0])
        rew[:, :, t] = r
        ret += r
    return states, obs, act, rew, ret


def _write(out, episodes_out, totals_out, states_out, obs_out, actions_out, rewards_out, res, fitness):
    states, obs, act, rew, ret = res
    for t, v in ((states_out, states), (obs_out, obs), (actions_out, act), (rewards_out, rew)):
        if t is not None:
            t.copy_(torch.from_numpy(v).reshape(t.shape))
    if episodes_out is not None:
        episodes_out.copy_(torch.from_numpy(ret.astype(np.float32)).reshape(episodes_out.shape))
    if totals_out is not None:
        o = obs.astype(np.float64).reshape(-1, 3)
        totals_out.copy_(torch.from_numpy(np.concatenate([o.sum(0), (o * o).sum(0), [o.shape[0]]])))
    f = torch.from_numpy(fitness.astype(np.float32))
    if out is None:
        return f
    out.copy_(f.reshape(out.shape))
    return out


def _stats(obs_stats):
    if obs_stats is None:
        return None
    a = obs_stats.numpy()
    return a[:3], a[3:6], a[6]


def rollout_record(theta, *, env=0, hidden, horizon=200, repetitions=10, sigma, clip, action_noise_std=0.0, seed,
                   generation=0, state=None, member_offset=0, n_local, noiseless=False, mirrored=False, obs_stats=None,
                   totals_out=None, workspace=None, out=None, episodes_out=None, states_out=None, obs_out=None,
                   actions_out=None, rewards_out=None):
    gen = int(state[0]) if state is not None else int(generation)
    CALLS.append(dict(op='rollout_record', seed=seed, generation=gen, member_offset=member_offset, n_local=n_local,
                      noiseless=noiseless, mirrored=mirrored, sigma=sigma, action_noise_std=action_noise_std,
                      repetitions=repetitions, theta=theta.clone(),
                      obs_stats=None if obs_stats is None else obs_stats.clone()))
    assert not (mirrored and noiseless)
    P, n = theta.numel(), int(n_local)
    if noiseless:
        rows = np.tile(theta.numpy().reshape(1, P), (n, 1))
        resets = np.full(n, po.TEST_MEMBER)
    else:
        eps = (mo.noise_mirrored if mirrored else orc.noise)(seed, gen, member_offset, n, P)
        rows = orc.perturb(theta.numpy(), sigma, eps).reshape(n, P)
        resets = np.arange(member_offset, member_offset + n)
    res = _episodes(np.asarray(rows, np.float32), hidden, seed, gen, resets, member_offset, repetitions, horizon, clip,
                    action_noise_std, _stats(obs_stats))
    return _write(out, episodes_out, totals_out, states_out, obs_out, actions_out, rewards_out, res, res[4].mean(1))


def rollout_record_solutions(solutions, *, env=0, hidden, horizon=200, repetitions=10, clip, action_noise_std=0.0, seed,
                             generation=0, member_offset=0, obs_stats=None, totals_out=None, workspace=None, out=None,
                             episodes_out=None, states_out=None, obs_out=None, actions_out=None, rewards_out=None):
    CALLS.append(dict(op='rollout_record_solutions', seed=seed, generation=generation, member_offset=member_offset,
                      n_local=solutions.shape[0], action_noise_std=action_noise_std, repetitions=repetitions))
    n = solutions.shape[0]
    res = _episodes(solutions.numpy(), hidden, seed, generation, np.arange(member_offset, member_offset + n),
                    member_offset, repetitions, horizon, clip, action_noise_std, _stats(obs_stats))
    return _write(out, episodes_out, totals_out, states_out, obs_out, actions_out, rewards_out, res, res[4].mean(1))
