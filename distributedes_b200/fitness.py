"""Fitness sources, one per kind of environment: the tape (Tape), episodes stepped on the device (DeviceRollouts) and
episodes stepped on the host (HostRollouts).  engine.NESEngine and cma_es.Worker evaluate through one and never ask
which.  HostSweep is HostRollouts for every run of a sweep at once (engine.HostEnvSweepEngine, cma_es.SweepWorker), and
DeviceSweep DeviceRollouts' evaluation of explicit rows for every run of a CMA-ES sweep.  A source evaluates NES members
theta + sigma*eps (`members`) or explicit rows (`solutions`), runs test episodes,
holds the normaliser statistics `obs_stats` [m | v | n] (or None) and the fp64 observation totals `obs_totals` of its
last evaluation, shares and merges them over an engine.RankGroup, counts its environment steps and says whether a CUDA
graph may capture it.  from_config builds the source a config describes, for both trainers."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from .envs import TEST_MEMBER, DeviceEnv, GymEnvBatch

POLICY_WIDTHS = (16, 32, 64, 96, 128)     # hidden widths des_rollout_eval and des_policy_act take (H/16 units per lane)


class Tape:
    """Fitness on the observation tape.  NES members go through des_nes_eval (after des_obs_normalize of the tape with
    the statistics of the previous generations, when normalising); explicit rows through des_pop_eval on the raw tape.
    A tape without a `sigma` evaluates explicit rows only (CMA-ES), so it keeps no normaliser and no eval workspace.
    Every member sees the whole tape, so the statistics merge needs no collective."""

    test_repetitions = 1          # the tape is deterministic

    def __init__(self, kernels, device, obs, target, *, state_dim, hidden, action_dim, clip, repetitions=1,
                 normalize_obs=False, sigma=None, seed=0, precision='fp32', mirrored=False):
        self.k, self.device = kernels, torch.device(device)
        self.d0, self.H, self.A, self.clip = int(state_dim), int(hidden), int(action_dim), float(clip)
        self.repetitions, self.normalize_obs = int(repetitions), bool(normalize_obs) and sigma is not None
        self.sigma, self.seed, self.precision, self.mirrored = sigma, int(seed), precision, bool(mirrored)
        self.obs_stats = torch.zeros(2 * self.d0 + 1, dtype=torch.float32, device=self.device) if self.normalize_obs else None
        self.obs_totals = self.obs_raw = self.T = self.eval_ws = None
        self.set_tape(obs, target)

    def set_tape(self, obs, target):
        """Returns whether the buffers moved: a tape of the current shape is copied in place (stable for a graph)."""
        obs = torch.as_tensor(obs, dtype=torch.float32)
        target = torch.as_tensor(target, dtype=torch.float32)
        if obs.dim() != 2 or obs.shape[1] != self.d0 or target.dim() != 2 or target.shape[1] != self.A \
                or target.shape[0] != obs.shape[0]:
            raise ValueError('tape shapes %r / %r do not match (T,%d) / (T,%d)' %
                             (tuple(obs.shape), tuple(target.shape), self.d0, self.A))
        if self.obs_raw is not None and self.obs_raw.shape == obs.shape:
            self.obs_raw.copy_(obs, non_blocking=True)
            self.target.copy_(target, non_blocking=True)
            return False
        self.obs_raw = obs.to(self.device).contiguous()
        self.target = target.to(self.device).contiguous()
        # what the kernels read: the raw tape, or its normalised image refreshed every generation
        self.obs = torch.empty_like(self.obs_raw) if self.normalize_obs else self.obs_raw
        if int(obs.shape[0]) != self.T and self.sigma is not None and hasattr(self.k, 'eval_workspace'):
            # a new tape length may be a multi-pass tensor-core shape: size its tile cache for the new T
            self.eval_ws = self.k.eval_workspace(self.d0, self.H, self.A, int(obs.shape[0]), self.precision, self.device)
        self.T = int(obs.shape[0])
        return True

    def members(self, theta, *, state, generation, offset, n_local, out):
        if self.normalize_obs:        # utils.py:48-51 with the statistics of the previous generations
            self.k.obs_normalize(self.obs_raw, self.obs_stats, out=self.obs)
        if n_local:
            (self.k.nes_eval_mirrored if self.mirrored else self.k.nes_eval)(
                theta, self.obs, self.target, hidden=self.H, sigma=self.sigma, clip=self.clip, seed=self.seed,
                state=state, member_offset=offset, n_local=n_local, precision=self.precision, out=out,
                workspace=self.eval_ws)

    def solutions(self, solutions, *, offset, generation, out=None):
        return self.k.pop_eval(solutions, self.obs_raw, self.target, hidden=self.H, clip=self.clip, out=out)

    def test_returns(self, solution, repetitions, generation, state=None):
        """`repetitions` evaluations of one solution, one launch each as the reference's test() loops run them: NES's
        through the normaliser with des_nes_eval at sigma = 0, CMA-ES's (no sigma) as one row of des_pop_eval."""
        out = []
        for _ in range(repetitions):
            if self.sigma is None:
                f = self.solutions(solution.reshape(1, -1), offset=0, generation=generation)
            else:
                obs = self.k.obs_normalize(self.obs_raw, self.obs_stats) if self.normalize_obs else self.obs_raw
                f = self.k.nes_eval(solution, obs, self.target, hidden=self.H, sigma=0.0, clip=self.clip, seed=self.seed,
                                    generation=0, member_offset=0, n_local=1, precision='fp32')
            out.append(float(f[0]))
        return np.asarray(out)

    def share_totals(self, group):
        pass

    def merge(self, N):
        if self.normalize_obs:
            # natural_es.py:85-89: every member saw the whole tape, so every rank merges the same online statistics
            self.k.obs_stats_merge(self.obs_stats, self.obs_raw, N * self.T * self.repetitions)

    def steps(self, N, group):
        return N * self.repetitions * self.T

    def capturable(self, world):
        return True


class _Episodes:
    """The statistics of the states episodes visit: each rank sums its members' raw observations in fp64, and one
    (2*d0+1)-double all-reduce replaces the per-worker Chan merges of natural_es.py:85-89 / cma_es.py:92-96."""

    precision = 'fp32'            # the device policy of des_rollout_eval and des_policy_act

    def __init__(self, kernels, device, *, state_dim, hidden, clip, action_noise_std, seed, repetitions, normalize_obs,
                 sigma, mirrored):
        if int(hidden) not in POLICY_WIDTHS:
            raise ValueError('%s: hidden must be one of %s (the device policy keeps H/16 units per lane); got %r'
                             % (type(self).__name__, POLICY_WIDTHS, hidden))
        self.k, self.device = kernels, torch.device(device)
        self.d0, self.H, self.clip = int(state_dim), int(hidden), float(clip)
        self.action_noise_std, self.seed, self.repetitions = float(action_noise_std), int(seed), int(repetitions)
        self.normalize_obs, self.sigma, self.mirrored = bool(normalize_obs), sigma, bool(mirrored)
        w = 2 * self.d0 + 1
        self.obs_stats = torch.zeros(w, dtype=torch.float32, device=self.device) if self.normalize_obs else None
        self.obs_totals = torch.zeros(w, dtype=torch.float64, device=self.device)

    def set_tape(self, obs, target):
        raise TypeError('%s steps its environments; there is no tape to set' % type(self).__name__)

    def share_totals(self, group):
        if self.normalize_obs:
            group.sum_(self.obs_totals)

    def merge(self, N):
        if self.normalize_obs:
            self.k.obs_stats_merge_totals(self.obs_stats, self.obs_totals, self.d0)


class Trajectories(NamedTuple):
    """Recorded closed-loop episodes (DeviceRollouts.record): for each member, episode and step, row-major
    [members, repetitions, horizon, ...] (the surfaces that record test episodes drop the members axis):
    states fp64 [.., 2], gym's (th, thdot) before the step, th unwrapped; obs fp32 [.., d0], the raw observation the
    policy was given; actions fp32 [.., A], after action noise and the clip, before the environment's own clamp; rewards
    fp64 [..], what the step returned; returns fp32 [members, repetitions], the episode returns the evaluation writes,
    each the fp32 of the fp64 sum of its rewards in step order."""
    states: np.ndarray
    obs: np.ndarray
    actions: np.ndarray
    rewards: np.ndarray
    returns: np.ndarray

    def episode(self, i):
        """The trajectories of member i (a test recording's one member)."""
        return Trajectories(*(x[i] for x in self))


class DeviceRollouts(_Episodes):
    """Closed-loop episodes stepped on the device (SURVEY 8f row 3): Evaluator.eval utils.py:116-124 runs `repetitions`
    episodes per member, every member seeing its own observations.  Environment: a DeviceEnv task."""

    def __init__(self, kernels, device, *, task, hidden, repetitions, clip=None, horizon=None, **kw):
        if task not in DeviceEnv.SPECS:
            raise ValueError('closed-loop environments available on the device: %s (got %r)' % (sorted(DeviceEnv.SPECS), task))
        if not (1 <= int(repetitions) <= 10):
            raise ValueError('DeviceRollouts: repetitions must be in [1, 10] (one warp steps them in lockstep); got %r'
                             % (repetitions,))
        spec = DeviceEnv.SPECS[task]
        super().__init__(kernels, device, state_dim=spec['state_dim'], hidden=hidden,
                         clip=spec['clip'] if clip is None else clip, repetitions=repetitions, **kw)
        self.env_id, self.A, self.horizon = spec['env'], spec['action_dim'], int(horizon or spec['horizon'])
        self.T, self.test_repetitions = self.horizon, self.repetitions
        self.roll_ws = None

    def _workspace(self, n):
        w = 2 * self.d0 + 1
        if self.roll_ws is None or self.roll_ws.numel() < n * w:
            self.roll_ws = torch.empty(n * w, dtype=torch.float64, device=self.device)
        return self.roll_ws

    def _env(self):
        return dict(env=self.env_id, hidden=self.H, horizon=self.horizon, clip=self.clip,
                    action_noise_std=self.action_noise_std, seed=self.seed)

    def members(self, theta, *, state, generation, offset, n_local, out, bc_out=None):
        """Fitness of members [offset, offset + n_local) into out; with bc_out [n_local, d0], also their behaviours
        (des_rollout_eval_bc: the same fitness, bit for bit).  Behaviours of mirrored members are refused."""
        if bc_out is not None and self.mirrored:
            raise ValueError('DeviceRollouts: behaviours (bc_out) are written for plain members only; this source samples '
                             'mirrored pairs')
        self.obs_totals.zero_()
        if n_local:
            kw = dict(repetitions=self.repetitions, sigma=self.sigma, state=state, member_offset=offset, n_local=n_local,
                      obs_stats=self.obs_stats, totals_out=self.obs_totals if self.normalize_obs else None,
                      workspace=self._workspace(n_local), out=out, **self._env())
            if bc_out is not None:
                self.k.rollout_eval_bc(theta, bc_out=bc_out, **kw)
            else:
                (self.k.rollout_eval_mirrored if self.mirrored else self.k.rollout_eval)(theta, **kw)

    def solutions(self, solutions, *, offset, generation, out=None):
        n = int(solutions.shape[0])
        self.obs_totals.zero_()
        out = out if out is not None else torch.zeros(n, dtype=torch.float32, device=self.device)
        if n:
            self.k.rollout_eval_solutions(solutions, repetitions=self.repetitions, generation=generation,
                                          member_offset=offset, obs_stats=self.obs_stats,
                                          totals_out=self.obs_totals if self.normalize_obs else None,
                                          workspace=self._workspace(n), out=out, **self._env())
        return out

    def ga_members(self, parents, n_elites, generation, offset, n_local, out, bc_out=None):
        """The genetic algorithm's members [offset, offset + n_local) of `generation`, whose table is parents[T_g, P]
        with n_elites elites, evaluated by des_rollout_eval_ga: solutions() of genetic.GeneticAlgorithm.ask()'s rows, bit
        for bit, with each member's weights built on the device.  The sigma is this source's.  With bc_out [n_local, d0],
        also their behaviours (des_rollout_eval_ga_bc: the same fitness, bit for bit)."""
        self.obs_totals.zero_()
        if n_local:
            kw = dict(repetitions=self.repetitions, sigma=self.sigma, generation=generation, member_offset=offset,
                      n_local=n_local, obs_stats=self.obs_stats,
                      totals_out=self.obs_totals if self.normalize_obs else None, workspace=self._workspace(n_local),
                      out=out, **self._env())
            if bc_out is not None:
                self.k.rollout_eval_ga_bc(parents, n_elites, bc_out=bc_out, **kw)
            else:
                self.k.rollout_eval_ga(parents, n_elites, **kw)
        return out

    def test_returns(self, solution, repetitions, generation, state=None, bc_out=None):
        """Noiseless episodes from the test stream, keyed by the generation word in `state` if given, else `generation`;
        with bc_out [1, d0], the same launch writes the solution's behaviour (des_rollout_eval_bc)."""
        sol = solution.reshape(-1).to(device=self.device, dtype=torch.float32).contiguous()
        episodes = torch.empty(int(repetitions), dtype=torch.float32, device=self.device)
        word = dict(state=state) if state is not None else dict(generation=generation)
        kw = dict(repetitions=int(repetitions), sigma=0.0, member_offset=0, n_local=1, noiseless=True,
                  obs_stats=self.obs_stats, episodes_out=episodes, **word, **self._env())
        if bc_out is not None:
            self.k.rollout_eval_bc(sol, bc_out=bc_out, **kw)
        else:
            self.k.rollout_eval(sol, **kw)
        return episodes.cpu().numpy().astype(np.float64)

    def record(self, weights, *, repetitions=None, noiseless=False, state=None, generation=0, member_offset=0,
               n_local=1):
        """Trajectories of the episodes an evaluation runs, from one des_rollout_record[_solutions] launch with this
        source's statistics: explicit rows weights[n, P] as solutions() evaluates them, or members [member_offset,
        member_offset + n_local) of theta as members() does (noiseless: test episodes as test_returns() runs them, keyed
        by the generation word in `state` if given, else `generation`).  Reads the statistics and writes nothing else:
        obs_totals stay as they are."""
        reps, T, dev = int(repetitions or self.repetitions), self.horizon, self.device
        rows = weights.dim() == 2
        n = int(weights.shape[0]) if rows else int(n_local)
        f32, f64 = torch.float32, torch.float64
        traj = dict(states_out=torch.empty((n, reps, T, 2), dtype=f64, device=dev),
                    obs_out=torch.empty((n, reps, T, self.d0), dtype=f32, device=dev),
                    actions_out=torch.empty((n, reps, T, self.A), dtype=f32, device=dev),
                    rewards_out=torch.empty((n, reps, T), dtype=f64, device=dev))
        episodes = torch.empty((n, reps), dtype=f32, device=dev)
        if rows:
            self.k.rollout_record_solutions(weights, repetitions=reps, generation=generation, member_offset=member_offset,
                                            obs_stats=self.obs_stats, episodes_out=episodes, **traj, **self._env())
        else:
            word = dict(state=state) if state is not None else dict(generation=generation)
            theta = weights.reshape(-1).to(device=dev, dtype=f32).contiguous()
            self.k.rollout_record(theta, repetitions=reps, sigma=0.0 if noiseless else self.sigma,
                                  mirrored=self.mirrored and not noiseless, member_offset=member_offset, n_local=n,
                                  noiseless=noiseless, obs_stats=self.obs_stats, episodes_out=episodes, **word, **traj,
                                  **self._env())
        return Trajectories(*(traj[k].cpu().numpy() for k in ('states_out', 'obs_out', 'actions_out', 'rewards_out')),
                            returns=episodes.cpu().numpy())

    def steps(self, N, group):
        return N * self.repetitions * self.horizon

    def capturable(self, world):
        return world == 1 or not self.normalize_obs      # sharded, the observation totals travel through NCCL


def behaviour(final_obs):
    """[n, d0] fp32 behaviours from final_obs [n, repetitions, d0] fp32: each member's fp64 sum in episode order over
    its episodes, divided by the repetitions (des_rollout_eval_bc's contract, on the host)."""
    s = np.zeros(final_obs.shape[::2], dtype=np.float64)
    for r in range(final_obs.shape[1]):
        s += final_obs[:, r].astype(np.float64)
    return (s / final_obs.shape[1]).astype(np.float32)


class HostEpisodes:
    """The bridge between environments stepped on the host and the population's policy on the device: runs the episodes
    of `n` weight rows x `repetitions` in lockstep until every slot is done (Evaluator.eval / single_run,
    utils.py:116-139).  Per step: observations -> pinned buffer -> device, des_policy_act, actions -> host, env.step,
    fp64 return accumulation per slot.  Slot b = i * repetitions + r of the batch environment is episode r of row i.

    `batch_env` implements the protocol of envs.py (num_envs, reset(keys), step(actions, alive)); its num_envs must be
    n * repetitions."""

    def __init__(self, kernels, device, batch_env, n, repetitions, state_dim, hidden, action_dim, clip, action_noise_std,
                 seed):
        self.k, self.device, self.env = kernels, torch.device(device), batch_env
        self.n, self.reps = int(n), int(repetitions)
        self.d0, self.H, self.A = int(state_dim), int(hidden), int(action_dim)
        self.clip, self.action_noise_std, self.seed = float(clip), float(action_noise_std), int(seed)
        B = self.n * self.reps
        if int(batch_env.num_envs) != B:
            raise ValueError('the batch environment has %d slots; %d members x %d repetitions need %d'
                             % (batch_env.num_envs, self.n, self.reps, B))
        pin = self.device.type == 'cuda'
        self.obs_h = torch.empty((B, self.d0), dtype=torch.float32, pin_memory=pin)
        self.alive_h = torch.empty(B, dtype=torch.uint8, pin_memory=pin)
        self.act_h = torch.empty((B, self.A), dtype=torch.float32, pin_memory=pin)
        self.obs_d = torch.empty((B, self.d0), dtype=torch.float32, device=self.device)
        self.alive_d = torch.empty(B, dtype=torch.uint8, device=self.device)
        self.act_d = torch.empty((B, self.A), dtype=torch.float32, device=self.device)

    def run(self, rows, *, generation, member_offset=0, key_member=None, obs_stats=None, stat_part=None, final_obs=None):
        """Returns (returns[n, repetitions] fp64, environment steps taken).  Episode (i, r) resets with the key
        (generation, member_offset + i, r), or (generation, key_member, r) when key_member is given (test episodes,
        whose action noise then uses member 0 as des_rollout_eval's test episodes do).  final_obs, an fp32 array
        [n, repetitions, d0], receives the observation returned by the step that ended each episode."""
        n, reps, B = self.n, self.reps, self.n * self.reps
        if B == 0:
            return np.zeros((n, reps)), 0
        members = (np.full(n, int(key_member), dtype=np.int64) if key_member is not None
                   else int(member_offset) + np.arange(n, dtype=np.int64))
        keys = np.stack([np.full(B, int(generation) & 0xFFFFFFFF, dtype=np.int64), np.repeat(members, reps),
                         np.tile(np.arange(reps, dtype=np.int64), n)], axis=1)
        noise_offset = 0 if key_member is not None else int(member_offset)
        obs = self.env.reset(keys)
        alive = np.ones(B, dtype=bool)
        returns = np.zeros(B, dtype=np.float64)
        steps, t = 0, 0
        cuda = self.device.type == 'cuda'
        obs_h, alive_h, act_h = self.obs_h.numpy(), self.alive_h.numpy(), self.act_h.numpy()
        while alive.any():
            obs_h[:] = obs                                              # fp32 cast: FloatTensor(o), utils.py:42-45
            alive_h[:] = alive
            self.obs_d.copy_(self.obs_h, non_blocking=True)
            self.alive_d.copy_(self.alive_h, non_blocking=True)
            self.k.policy_act(rows, self.obs_d, self.alive_d, state_dim=self.d0, hidden=self.H, action_dim=self.A,
                              repetitions=reps, clip=self.clip, action_noise_std=self.action_noise_std, seed=self.seed,
                              generation=generation, member_offset=noise_offset, t=t, obs_stats=obs_stats,
                              stat_part=stat_part, out=self.act_d)
            self.act_h.copy_(self.act_d, non_blocking=True)
            if cuda:
                torch.cuda.current_stream(self.device).synchronize()
            obs, reward, done = self.env.step(act_h, alive)
            returns[alive] += np.asarray(reward, dtype=np.float64)[alive]      # utils.py:137
            steps += int(alive.sum())
            if final_obs is not None:
                ended = alive & np.asarray(done, dtype=bool)
                final_obs.reshape(B, self.d0)[ended] = np.asarray(obs, dtype=np.float32).reshape(B, self.d0)[ended]
            alive &= ~np.asarray(done, dtype=bool)
            t += 1
        return returns.reshape(n, reps), steps


class HostRollouts(_Episodes):
    """Episodes stepped on the HOST by the user's own code, the per-step policy on the device (des_policy_act):
    Evaluator.eval utils.py:116-124.  NES members become rows theta + sigma*eps once per generation (des_nes_perturb,
    natural_es.py:28-30).  The step count is the episodes' real length, summed over ranks (natural_es.py:75,
    cma_es.py:73).  batch_env_fn(num_slots) builds a batch environment (envs.py); the default wraps env_fn in
    envs.GymEnvBatch.  env_fn is probed for the dimensions when they are not given."""

    def __init__(self, kernels, device, *, env_fn, hidden, repetitions, state_dim=None, action_dim=None,
                 test_repetitions=None, batch_env_fn=None, **kw):
        if state_dim is None or action_dim is None:
            probe = env_fn()
            state_dim, action_dim = probe.observation_space.shape[0], probe.action_space.shape[0]
        if not (1 <= int(state_dim) <= 32 and 1 <= int(action_dim) <= 8):
            raise ValueError('HostRollouts: des_policy_act takes state_dim <= 32 and action_dim <= 8; got %r, %r'
                             % (state_dim, action_dim))
        for name, r in (('repetitions', repetitions), ('test_repetitions', test_repetitions or repetitions)):
            if not (1 <= int(r) <= 16):
                raise ValueError('HostRollouts: %s must be in [1, 16]; got %r' % (name, r))
        super().__init__(kernels, device, state_dim=state_dim, hidden=hidden, repetitions=repetitions, **kw)
        self.A, self.test_repetitions = int(action_dim), int(test_repetitions or repetitions)
        if batch_env_fn is None:
            batch_env_fn = lambda B: GymEnvBatch(env_fn, B, self.seed)      # noqa: E731
        self.batch_env_fn = batch_env_fn
        self._bridges = {}            # (rows, repetitions) -> HostEpisodes
        self.rows = self.stat_part = None
        self.last_steps = 0           # environment steps of the last evaluation on this rank

    def _bridge(self, n, reps):
        ep = self._bridges.get((n, reps))
        if ep is None:
            ep = HostEpisodes(self.k, self.device, self.batch_env_fn(n * reps), n, reps, self.d0, self.H, self.A,
                              self.clip, self.action_noise_std, self.seed)
            self._bridges[(n, reps)] = ep
        return ep

    def members(self, theta, *, state, generation, offset, n_local, out, bc_out=None):
        """Fitness of members [offset, offset + n_local) into out; with bc_out [n_local, d0], also their behaviours: each
        member's observations after its episodes' last steps, averaged over the repetitions (behaviour()).  Mirrored
        members have them too: their rows are the mirrored perturbations."""
        self.obs_totals.zero_()
        self.last_steps = 0
        if n_local:
            if self.rows is None:
                self.rows = torch.empty((n_local, theta.numel()), dtype=torch.float32, device=self.device)
            (self.k.nes_perturb_mirrored if self.mirrored else self.k.nes_perturb)(theta, n_local, self.sigma, self.seed, generation,
                                                      member_offset=offset, out=self.rows)
            self._episodes(self.rows, offset, generation, out, bc_out)

    def solutions(self, solutions, *, offset, generation, out=None, bc_out=None):
        """Fitness of explicit rows solutions[n, P] as members offset.. into out; with bc_out [n, d0], also their
        behaviours from the same episodes (behaviour())."""
        n = int(solutions.shape[0])
        self.obs_totals.zero_()
        self.last_steps = 0
        out = out if out is not None else torch.zeros(n, dtype=torch.float32, device=self.device)
        if n:
            self._episodes(solutions.to(device=self.device, dtype=torch.float32).contiguous(), offset, generation, out,
                           bc_out)
        return out

    def _episodes(self, rows, offset, generation, out, bc_out=None):
        n = int(rows.shape[0])
        if self.stat_part is None or self.stat_part.shape[0] != n:
            self.stat_part = torch.zeros((n, 2 * self.d0 + 1), dtype=torch.float64, device=self.device)
        else:
            self.stat_part.zero_()
        part = self.stat_part if self.normalize_obs else None
        final = None if bc_out is None else np.zeros((n, self.repetitions, self.d0), dtype=np.float32)
        ret, self.last_steps = self._bridge(n, self.repetitions).run(rows, generation=generation, member_offset=offset,
                                                                     obs_stats=self.obs_stats, stat_part=part,
                                                                     final_obs=final)
        out.copy_(torch.from_numpy(ret.mean(axis=1).astype(np.float32)))       # -cost, utils.py:124
        if part is not None:
            self.k.obs_parts_reduce(part, self.d0, out=self.obs_totals)
        if bc_out is not None:
            bc_out.copy_(torch.from_numpy(behaviour(final)).reshape(bc_out.shape))

    def test_returns(self, solution, repetitions, generation, state=None, bc_out=None):
        """Episodes keyed (generation, TEST_MEMBER, repetition), which do not feed the statistics; `state` is not read.
        With bc_out [1, d0], also the solution's behaviour from the same episodes."""
        row = solution.reshape(1, -1).to(device=self.device, dtype=torch.float32).contiguous()
        final = None if bc_out is None else np.zeros((1, int(repetitions), self.d0), dtype=np.float32)
        ret, _ = self._bridge(1, int(repetitions)).run(row, generation=generation, key_member=TEST_MEMBER,
                                                       obs_stats=self.obs_stats, final_obs=final)
        if bc_out is not None:
            bc_out.copy_(torch.from_numpy(behaviour(final)).reshape(bc_out.shape))
        return ret[0]

    def steps(self, N, group):
        return int(group.sum_(torch.tensor([self.last_steps], dtype=torch.int64, device=self.device)).item())

    def capturable(self, world):
        return False


class HostSweepEpisodes:
    """HostEpisodes for every run of a sweep in lockstep.  envs[r] is run r's batch environment of n * repetitions slots
    and rows r*n .. r*n + n - 1 of the weights are its members (ops_sweep: member_offset 0 under run r's seed).  Per step:
    every slot's observations and alive flags to the device in one copy each, one des_policy_act_sweep, the actions back in
    one copy and one synchronise, then step(actions_r, alive_r) of every run that still has an alive slot.  So each run's
    environment receives exactly the reset and step calls its standalone HostEpisodes makes.  The runs `running` leaves
    out are neither reset nor stepped: their slots enter every launch dead."""

    def __init__(self, kernels, device, envs, n, repetitions, state_dim, hidden, action_dim, clip):
        self.k, self.device, self.envs = kernels, torch.device(device), list(envs)
        self.R, self.n, self.reps = len(self.envs), int(n), int(repetitions)
        self.d0, self.H, self.A, self.clip = int(state_dim), int(hidden), int(action_dim), float(clip)
        B = self.n * self.reps
        for r, env in enumerate(self.envs):
            if int(env.num_envs) != B:
                raise ValueError('run %d: the batch environment has %d slots; %d members x %d repetitions need %d'
                                 % (r, env.num_envs, self.n, self.reps, B))
        pin, RB = self.device.type == 'cuda', self.R * B
        self.obs_h = torch.zeros((RB, self.d0), dtype=torch.float32, pin_memory=pin)
        self.alive_h = torch.zeros(RB, dtype=torch.uint8, pin_memory=pin)
        self.act_h = torch.zeros((RB, self.A), dtype=torch.float32, pin_memory=pin)
        self.obs_d = torch.zeros((RB, self.d0), dtype=torch.float32, device=self.device)
        self.alive_d = torch.zeros(RB, dtype=torch.uint8, device=self.device)
        self.act_d = torch.zeros((RB, self.A), dtype=torch.float32, device=self.device)

    def run(self, rows, hp, *, generation, running, key_member=None, obs_stats=None, stat_part=None, final_obs=None):
        """Returns (returns[R, n, repetitions] fp64, environment steps[R]); the runs not `running` return zeros.  The
        episodes' keys are HostEpisodes.run's at member_offset 0, the same for every run (each env seeds with its run's
        seed).  final_obs, an fp32 array [R, n, repetitions, d0], receives the observation returned by the step that
        ended each episode, as HostEpisodes.run's does; the slots of runs not `running` are left as they are."""
        R, n, reps, B, d0 = self.R, self.n, self.reps, self.n * self.reps, self.d0
        members = (np.full(n, int(key_member), dtype=np.int64) if key_member is not None else np.arange(n, dtype=np.int64))
        keys = np.stack([np.full(B, int(generation) & 0xFFFFFFFF, dtype=np.int64), np.repeat(members, reps),
                         np.tile(np.arange(reps, dtype=np.int64), n)], axis=1)
        returns, reward, done = (np.zeros((R, B), dtype=np.float64), np.zeros((R, B)), np.zeros((R, B), dtype=bool))
        steps = np.zeros(R, dtype=np.int64)
        alive = np.zeros((R, B), dtype=bool)
        obs_h = self.obs_h.numpy().reshape(R, B, d0)
        alive_h, act_h = self.alive_h.numpy().reshape(R, B), self.act_h.numpy().reshape(R, B, self.A)
        for r in np.flatnonzero(running):
            obs_h[r] = self.envs[r].reset(keys.copy())                # fp32 cast: FloatTensor(o), utils.py:42-45
            alive[r] = True
        cuda, t = self.device.type == 'cuda', 0
        while alive.any():
            alive_h[:] = alive
            self.obs_d.copy_(self.obs_h, non_blocking=True)
            self.alive_d.copy_(self.alive_h, non_blocking=True)
            self.k.policy_act_sweep(rows, self.obs_d, self.alive_d, hp, state_dim=d0, hidden=self.H, action_dim=self.A,
                                    repetitions=reps, clip=self.clip, generation=generation, run_size=n, t=t,
                                    obs_stats=obs_stats, stat_part=stat_part, out=self.act_d)
            self.act_h.copy_(self.act_d, non_blocking=True)
            if cuda:
                torch.cuda.current_stream(self.device).synchronize()
            for r in np.flatnonzero(alive.any(axis=1)):
                obs_h[r], reward[r], done[r] = self.envs[r].step(act_h[r], alive[r])
            np.add(returns, reward, out=returns, where=alive)                   # utils.py:137, alive slots only
            steps += alive.sum(axis=1)
            if final_obs is not None:
                ended = alive & done
                final_obs.reshape(R, B, d0)[ended] = obs_h[ended]
            alive &= ~done
            t += 1
        return returns.reshape(R, n, reps), steps


class HostSweep:
    """Episodes stepped on the host for every run of a sweep (engine.HostEnvSweepEngine): run r is the HostRollouts of its
    own environment factories, seed, sigma and action noise, at member_offset 0, and all runs step in lockstep through
    HostSweepEpisodes.  `runs` holds one dict per run with env_fn, batch_env_fn (None: envs.GymEnvBatch of env_fn under
    the run's seed), seed, sigma and action_noise_std; the rest is shared.  Owns each run's batch environments (built as
    HostRollouts builds them: batch_env_fn(N * repetitions) for the members, batch_env_fn(test_repetitions) for the test
    episodes), the pinned and device buffers of the bridges, the weight rows [R * N, P], stat_part [R * N, 2*d0+1], the
    statistics obs_stats and the observation totals obs_totals [R, 2*d0+1]."""

    def __init__(self, kernels, device, *, runs, hidden, repetitions, clip, normalize_obs, state_dim=None,
                 action_dim=None, test_repetitions=None):
        self.k, self.device = kernels, torch.device(device)
        self.runs = [HostRollouts(kernels, device, hidden=hidden, repetitions=repetitions, state_dim=state_dim,
                                  action_dim=action_dim, test_repetitions=test_repetitions, clip=clip,
                                  normalize_obs=normalize_obs, mirrored=False, **run) for run in runs]
        src = self.runs[0]
        for r, x in enumerate(self.runs):
            if (x.d0, x.A) != (src.d0, src.A):
                raise ValueError('HostSweep: run %d\'s environment has state_dim %d and action_dim %d; run 0\'s has %d '
                                 'and %d' % (r, x.d0, x.A, src.d0, src.A))
        self.R, self.d0, self.H, self.A, self.clip = len(self.runs), src.d0, src.H, src.A, src.clip
        self.repetitions, self.test_repetitions, self.normalize_obs = src.repetitions, src.test_repetitions, src.normalize_obs
        w = 2 * self.d0 + 1
        self.obs_stats = torch.zeros((self.R, w), dtype=torch.float32, device=self.device) if self.normalize_obs else None
        self.obs_totals = torch.zeros((self.R, w), dtype=torch.float64, device=self.device)
        self._bridges = {}            # (rows per run, repetitions) -> HostSweepEpisodes
        self.rows = self.stat_part = None
        self.last_steps = np.zeros(self.R, dtype=np.int64)

    def _bridge(self, n, reps):
        ep = self._bridges.get((n, reps))
        if ep is None:
            ep = HostSweepEpisodes(self.k, self.device, [x.batch_env_fn(n * reps) for x in self.runs], n, reps, self.d0,
                                   self.H, self.A, self.clip)
            self._bridges[(n, reps)] = ep
        return ep

    def members(self, theta, hp, *, generation, run_size, running, out, bc_out=None):
        """fitness out[R, N] of every run's members theta_r + sigma_r eps (one des_nes_perturb_sweep), its steps in
        last_steps and, normalising, its observation totals in obs_totals.  With bc_out [R, N, d0], also their behaviours:
        HostRollouts.members' of every running run (behaviour())."""
        N = int(run_size)
        if self.rows is None:
            self.rows = torch.empty((self.R * N, theta.shape[1]), dtype=torch.float32, device=self.device)
        self.k.nes_perturb_sweep(theta, hp, N, generation, out=self.rows)
        self._episodes(self.rows, hp, N, generation, running, out, bc_out)

    def solutions(self, rows, hp, *, generation, running, out):
        """members without the perturbation (CMA-ES): rows [R * N, P] are every run's explicit solutions, run r's N rows
        r*N .. r*N + N - 1 of them, evaluated as HostRollouts.solutions evaluates one run's at offset 0."""
        self._episodes(rows, hp, rows.shape[0] // self.R, generation, running, out)

    def _episodes(self, rows, hp, N, generation, running, out, bc_out=None):
        w = 2 * self.d0 + 1
        self.obs_totals.zero_()
        if self.stat_part is None or self.stat_part.shape[0] != self.R * N:
            self.stat_part = torch.zeros((self.R * N, w), dtype=torch.float64, device=self.device)
        else:
            self.stat_part.zero_()
        part = self.stat_part if self.normalize_obs else None
        final = None if bc_out is None else np.zeros((self.R, N, self.repetitions, self.d0), dtype=np.float32)
        ret, self.last_steps = self._bridge(N, self.repetitions).run(rows, hp, generation=generation,
                                                                     running=running, obs_stats=self.obs_stats,
                                                                     stat_part=part, final_obs=final)
        out.copy_(torch.from_numpy(np.stack([ret[r].mean(axis=1).astype(np.float32) for r in range(self.R)])))
        if part is not None:
            self.k.obs_parts_reduce_runs(part, self.d0, N, out=self.obs_totals)
        if bc_out is not None:
            self._behaviours(final, bc_out)

    def _behaviours(self, final, bc_out):
        """bc_out [R, n, d0] from the final observations [R, n, repetitions, d0] (behaviour())."""
        R, n, reps, d0 = final.shape
        bc_out.copy_(torch.from_numpy(behaviour(final.reshape(R * n, reps, d0))).reshape(bc_out.shape))

    def test_returns(self, theta, hp, repetitions, generation, running, bc_out=None):
        """[R, repetitions] fp64: every running run's episodes keyed (generation, TEST_MEMBER, repetition) of theta[r]
        with its statistics, as HostRollouts.test_returns; they do not feed the statistics.  With bc_out [R, 1, d0],
        also every running run's behaviour from the same episodes."""
        final = None if bc_out is None else np.zeros((self.R, 1, int(repetitions), self.d0), dtype=np.float32)
        ret, _ = self._bridge(1, int(repetitions)).run(theta, hp, generation=generation, running=running,
                                                       key_member=TEST_MEMBER, obs_stats=self.obs_stats,
                                                       final_obs=final)
        if bc_out is not None:
            self._behaviours(final, bc_out)
        return ret[:, 0]


class DeviceSweep:
    """DeviceRollouts.solutions for every run of a CMA-ES sweep (cma_es.SweepWorker): run r is the DeviceRollouts of its
    own seed and action noise evaluating its rows at offset 0, all runs in one des_rollout_eval_solutions_sweep per
    generation and their test episodes in one noiseless des_rollout_eval_sweep.  The seeds and action noise are the rows
    of the sweep table `hp` the caller passes; the rest is shared.  Holds the statistics obs_stats and the observation
    totals obs_totals [R, 2*d0+1]."""

    def __init__(self, kernels, device, *, runs, task, hidden, repetitions, clip=None, normalize_obs, horizon=None):
        one = DeviceRollouts(kernels, device, task=task, hidden=hidden, repetitions=repetitions, clip=clip,
                             horizon=horizon, action_noise_std=0.0, seed=0, normalize_obs=normalize_obs, sigma=None,
                             mirrored=False)                      # the checks and the shared settings of every run
        self.k, self.device, self.R = kernels, one.device, int(runs)
        self.d0, self.H, self.A, self.clip, self.env_id, self.horizon = one.d0, one.H, one.A, one.clip, one.env_id, one.horizon
        self.repetitions, self.test_repetitions, self.normalize_obs = one.repetitions, one.test_repetitions, one.normalize_obs
        w = 2 * self.d0 + 1
        self.obs_stats = torch.zeros((self.R, w), dtype=torch.float32, device=self.device) if self.normalize_obs else None
        self.obs_totals = torch.zeros((self.R, w), dtype=torch.float64, device=self.device)
        self.roll_ws = self.fitness = None

    def _env(self):
        return dict(env=self.env_id, hidden=self.H, horizon=self.horizon, clip=self.clip)

    def solutions(self, rows, hp, *, generation, running, out):
        """fitness out[R, N] of every run's rows [R * N, P] (run r's N rows r*N ..), and, normalising, each run's
        observation totals in obs_totals.  Closed-loop runs stop together: `running` is not read."""
        N, w = rows.shape[0] // self.R, 2 * self.d0 + 1
        if self.roll_ws is None or self.roll_ws.numel() < self.R * N * w:
            self.roll_ws = torch.empty(self.R * N * w, dtype=torch.float64, device=self.device)
        self.obs_totals.zero_()
        self.k.rollout_eval_solutions_sweep(rows, hp, repetitions=self.repetitions, generation=generation, run_size=N,
                                            obs_stats=self.obs_stats,
                                            totals_out=self.obs_totals if self.normalize_obs else None,
                                            workspace=self.roll_ws, out=out, **self._env())

    def ga_members(self, parents, ga, hp, *, generation, out):
        """fitness out[R, N] of every genetic-algorithm run's generation, whose tables are parents[R, table_rows, P] with
        the counts of the table `ga` (des_rollout_eval_ga_sweep: each member's weights built on the device), and,
        normalising, each run's observation totals in obs_totals: DeviceRollouts.ga_members of every run under its seed,
        sigma and action noise, at offset 0."""
        N, w = out.shape[1], 2 * self.d0 + 1
        if self.roll_ws is None or self.roll_ws.numel() < self.R * N * w:
            self.roll_ws = torch.empty(self.R * N * w, dtype=torch.float64, device=self.device)
        self.obs_totals.zero_()
        self.k.rollout_eval_ga_sweep(parents, ga, hp, repetitions=self.repetitions, generation=generation, run_size=N,
                                     obs_stats=self.obs_stats, totals_out=self.obs_totals if self.normalize_obs else None,
                                     workspace=self.roll_ws, out=out, **self._env())
        return out

    def test_returns(self, theta, hp, repetitions, generation, running):
        """[R, repetitions] fp64: run r's noiseless episodes of theta[r] from the test stream keyed by `generation`, with
        its statistics: DeviceRollouts.test_returns under run r's seed and action noise."""
        reps = int(repetitions)
        if self.fitness is None:
            self.fitness = torch.empty((self.R, 1), dtype=torch.float32, device=self.device)
        episodes = torch.empty((self.R, 1, reps), dtype=torch.float32, device=self.device)
        self.k.rollout_eval_sweep(theta, hp, repetitions=reps, generation=generation, run_size=1, noiseless=True,
                                  obs_stats=self.obs_stats, out=self.fitness, episodes_out=episodes, **self._env())
        return episodes.reshape(self.R, reps).cpu().numpy().astype(np.float64)

    def steps(self, N):
        """[R] environment steps of the last evaluation: every episode runs its whole horizon."""
        return np.full(self.R, N * self.repetitions * self.horizon, dtype=np.int64)


def from_config(config, kernels, device, *, sigma=None, mirrored=False):
    """The source a config describes, for either trainer: `host_env` configs step on the host, `closed_loop` ones on the
    device, the rest read the tape of config.env_fn().  `sigma` and `mirrored` are NES's sampling of members; without a
    sigma the source evaluates explicit rows (CMA-ES)."""
    kw = dict(hidden=config.hidden_size, clip=config.clip, seed=config.seed, repetitions=config.repetitions,
              normalize_obs=config.normalize_obs, sigma=sigma, mirrored=mirrored)
    if getattr(config, 'host_env', False):
        return HostRollouts(kernels, device, env_fn=config.env_fn, batch_env_fn=getattr(config, 'batch_env_fn', None),
                            state_dim=config.state_dim, action_dim=config.action_dim,
                            test_repetitions=config.test_repetitions, action_noise_std=config.action_noise_std, **kw)
    if getattr(config, 'closed_loop', False):
        return DeviceRollouts(kernels, device, task=config.task, action_noise_std=config.action_noise_std, **kw)
    env = config.env_fn()
    return Tape(kernels, device, env.obs, env.target, state_dim=env.obs.shape[1], action_dim=env.target.shape[1],
                precision=config.precision, **kw)
