"""Per-GPU engine for the NES generation: the host logic around the CUDA kernels.

One process per GPU owns a contiguous shard of the population (the reference's Worker processes,
natural_es.py:10-32, each evaluate whatever task they pop; here member identity is fixed so noise can
be regenerated instead of shipped).  Per generation (natural_es.py:62-96):

    eval shard            des_nes_eval             -> fitness_all[off:off+n]   (zero elsewhere)
    [all-reduce fitness_all]   N floats; sum of zero-padded shards == all-gather, ragged shards allowed
    centered rank         des_centered_rank        -> shaped[n]   (global ranks of the local members)
    fitness x noise       des_nes_grad_partial     -> partial[P]
    [all-reduce partial]       P floats — the one collective BASELINE.json's north_star names
    (1-wd), Adam, step    des_nes_apply + des_state_advance   (identical on every rank: no broadcast)

`kernels` is the module providing the device ops (default: distributedes_b200.ops -> libdes_b200.so).
It exists so the world_size>1 host logic can be exercised on CPU with gloo by the test-suite, which
injects an oracle-backed stand-in; the product never runs without the CUDA library.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist


def shard_bounds(N, world_size, rank):
    """Contiguous split of N members over world_size ranks; the first N % world_size ranks get one more."""
    if world_size < 1 or not (0 <= rank < world_size):
        raise ValueError('bad rank %r / world_size %r' % (rank, world_size))
    base, rem = divmod(int(N), int(world_size))
    start = rank * base + min(rank, rem)
    return start, base + (1 if rank < rem else 0)


class NESEngine:
    def __init__(self, *, state_dim, hidden, action_dim, pop_size, theta0, obs, target, sigma, learning_rate,
                 weight_decay=0.005, clip=1.0, seed=0, precision='fp32', beta1=0.9, beta2=0.999, epsilon=1e-8,
                 device=None, process_group=None, kernels=None, use_graph=False, normalize_obs=False, repetitions=1,
                 mirrored=False):
        if kernels is None:
            from . import ops as kernels          # loads libdes_b200.so; raises if it is missing
        self.k = kernels
        self.pg = process_group
        distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(process_group) if distributed else 1
        self.rank = dist.get_rank(process_group) if distributed else 0
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        self.d0, self.H, self.A = int(state_dim), int(hidden), int(action_dim)
        self.N = int(pop_size)
        if self.N < 2:
            raise ValueError('pop_size must be >= 2 (fitness_shift divides by N-1, utils.py:146)')
        # mirrored sampling: members 2p and 2p+1 are theta +- sigma*eps_p; a shard holds whole pairs
        self.mirrored = bool(mirrored)
        if self.mirrored:
            if self.N % 2:
                raise ValueError('mirrored sampling needs an even pop_size (members come in +-eps pairs); got %d' % self.N)
            pair_offset, pairs = shard_bounds(self.N // 2, self.world, self.rank)
            self.offset, self.n_local = 2 * pair_offset, 2 * pairs
        else:
            self.offset, self.n_local = shard_bounds(self.N, self.world, self.rank)
        self.sigma, self.lr, self.wd, self.clip = float(sigma), float(learning_rate), float(weight_decay), float(clip)
        self.beta1, self.beta2, self.epsilon = float(beta1), float(beta2), float(epsilon)
        self.seed, self.precision = int(seed), precision
        theta0 = np.ascontiguousarray(theta0, dtype=np.float32).reshape(-1)
        self.P = self.k.param_count(self.d0, self.H, self.A)
        if theta0.size != self.P:
            raise ValueError('theta0 has %d entries, the (%d,%d,%d) MLP needs %d' %
                             (theta0.size, self.d0, self.H, self.A, self.P))
        dev = self.device
        self.theta = torch.from_numpy(theta0.copy()).to(dev)
        self.adam_m = torch.zeros(self.P, dtype=torch.float64, device=dev)
        self.adam_v = torch.zeros(self.P, dtype=torch.float64, device=dev)
        # sharded runs on the real library exchange fitness / partial sums through peer memory (comm.PeerComm: kernels of
        # this library storing over NVLink); DES_COMM=nccl (or a failure to map the peers) keeps the two NCCL all-reduces
        self.comm = None
        import os
        if self.world > 1 and kernels.__name__.endswith('.ops') and dev.type == 'cuda' and os.environ.get('DES_COMM', 'peer') != 'nccl':
            try:
                from .comm import PeerComm
                self.comm = PeerComm(self.N, self.P, dev, process_group)
            except RuntimeError as e:
                import warnings
                warnings.warn('distributedes_b200: peer-memory exchange unavailable (%s); using NCCL all-reduces' % e)
                self.comm = None
            # every rank must take the same path
            ok = torch.tensor([1 if self.comm is not None else 0], device=dev)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=process_group)
            if int(ok.item()) == 0 and self.comm is not None:
                self.comm.close()
                self.comm = None
        # fitness_all is PRIVATE to this rank: what callers read after generation().  With the peer-memory exchange the shard
        # is evaluated into the exchange block (which every peer writes its own range of — a peer that runs ahead may already
        # store the NEXT generation's shard there while this rank's host still reads this one) and the gathered vector is
        # copied out of it, stream-ordered, before any peer can get that far.
        self.fitness_all = torch.zeros(self.N, dtype=torch.float32, device=dev)
        self._fitness_xchg = self.comm.fitness_all if self.comm is not None else self.fitness_all
        self.partial_local = torch.zeros(self.P, dtype=torch.float32, device=dev) if self.comm is not None else None
        self.shaped = torch.zeros(max(self.n_local, 1), dtype=torch.float32, device=dev)[:self.n_local]
        self.partial = torch.zeros(self.P, dtype=torch.float32, device=dev)
        self.update = torch.zeros(self.P, dtype=torch.float32, device=dev)
        self.state = self.k.new_state(dev, 0)
        self.rank_ws = self.k.rank_workspace(self.n_local, dev, self.N)
        self.grad_ws = self.k.grad_workspace(self.n_local, self.P, dev)
        # observation normaliser (StaticNormalizer / SharedStats, utils.py:37-106): device-resident [m | v | n]
        self.normalize_obs = bool(normalize_obs)
        self.repetitions = int(repetitions)
        self.obs_stats = torch.zeros(2 * self.d0 + 1, dtype=torch.float32, device=dev) if self.normalize_obs else None
        self._setup_inputs(obs, target)
        self.generation_index = 0
        self._graph = None
        # the whole generation is one CUDA graph: always on a single GPU; sharded, when the exchange runs on the
        # peer-memory kernels (nothing but kernels of this library in the stream).  With NCCL collectives the generation
        # stays eager unless DES_GRAPH_NCCL=1 (capturing ProcessGroupNCCL collectives hung on the 2-GPU box in round 1).
        self._use_graph = (bool(use_graph) and self.device.type == 'cuda'
                           and (self.world == 1 or self.comm is not None or os.environ.get('DES_GRAPH_NCCL') == '1'))

    # -- inputs ------------------------------------------------------------------------------------------
    def _setup_inputs(self, obs, target):
        self.set_tape(obs, target)
        self.eval_ws = (self.k.eval_workspace(self.d0, self.H, self.A, self.T, self.precision, self.device)
                        if hasattr(self.k, 'eval_workspace') else None)

    def set_tape(self, obs, target):
        obs = torch.as_tensor(obs, dtype=torch.float32)
        target = torch.as_tensor(target, dtype=torch.float32)
        if obs.dim() != 2 or obs.shape[1] != self.d0 or target.dim() != 2 or target.shape[1] != self.A \
                or target.shape[0] != obs.shape[0]:
            raise ValueError('tape shapes %r / %r do not match (T,%d) / (T,%d)' %
                             (tuple(obs.shape), tuple(target.shape), self.d0, self.A))
        if getattr(self, 'obs_raw', None) is not None and self.obs_raw.shape == obs.shape:
            self.obs_raw.copy_(obs, non_blocking=True)      # keep addresses stable for a captured graph
            self.target.copy_(target, non_blocking=True)
        else:
            self.obs_raw = obs.to(self.device).contiguous()
            self.target = target.to(self.device).contiguous()
            # what the kernels read: the raw tape, or its normalised image refreshed every generation
            self.obs = torch.empty_like(self.obs_raw) if self.normalize_obs else self.obs_raw
            self._graph = None
            if getattr(self, 'T', None) is not None and int(obs.shape[0]) != self.T and hasattr(self.k, 'eval_workspace'):
                # a new tape length may be a multi-pass tensor-core shape: size its tile cache for the new T
                self.eval_ws = self.k.eval_workspace(self.d0, self.H, self.A, int(obs.shape[0]), self.precision, self.device)
        self.T = int(obs.shape[0])

    def _op(self, name):
        """The device op `name`, or its mirrored-noise counterpart when the engine samples mirrored pairs."""
        return getattr(self.k, name + '_mirrored' if self.mirrored else name)

    # -- the three phases around the two collectives -------------------------------------------------------
    def evaluate(self):
        if self.normalize_obs:        # utils.py:48-51 with the statistics of the previous generations
            self.k.obs_normalize(self.obs_raw, self.obs_stats, out=self.obs)
        if self.world > 1 and self.comm is None:
            self.fitness_all.zero_()
        if self.n_local:
            self._op('nes_eval')(self.theta, self.obs, self.target, hidden=self.H, sigma=self.sigma, clip=self.clip,
                            seed=self.seed, state=self.state, member_offset=self.offset, n_local=self.n_local,
                            precision=self.precision, out=self.fitness_shard_out,
                            workspace=self.eval_ws)
        self._gather_fitness()
        return self.fitness_all

    @property
    def fitness_shard_out(self):
        """Where this rank's evaluation kernel writes its shard (the exchange block when peers read it from there)."""
        return self._fitness_xchg[self.offset:self.offset + self.n_local]

    def _gather_fitness(self):
        if self.world > 1:
            if self.comm is not None:
                self.comm.allgather_fitness(self.offset, self.n_local)     # shard -> every peer's exchange block, flag barrier
                self.fitness_all.copy_(self._fitness_xchg)                 # the stable private copy (a 4N-byte device copy)
            else:
                dist.all_reduce(self.fitness_all, group=self.pg)

    def rank_and_reduce(self):
        self.k.centered_rank(self.fitness_all, self.offset, self.n_local, workspace=self.rank_ws, out=self.shaped)
        self._op('nes_grad_partial')(self.shaped, self.P, seed=self.seed, state=self.state, member_offset=self.offset,
                                     workspace=self.grad_ws,
                                     out=self.partial_local if self.comm is not None else self.partial)
        if self.world > 1:
            if self.comm is not None:
                self.comm.allreduce_partial(self.partial_local, self.partial)   # slots over NVLink, summed in rank order
            else:
                dist.all_reduce(self.partial, group=self.pg)
        return self.partial

    def apply(self):
        self.k.nes_apply(self.theta, self.adam_m, self.adam_v, self.partial, self.N, self.state, sigma=self.sigma,
                         learning_rate=self.lr, weight_decay=self.wd, beta1=self.beta1, beta2=self.beta2,
                         epsilon=self.epsilon, update_out=self.update)
        self.k.state_advance(self.state, self.beta1, self.beta2)
        self._merge_obs_stats()

    def _merge_obs_stats(self):
        if self.normalize_obs:
            # natural_es.py:85-89: merge this generation's online statistics (every member saw the whole tape;
            # all ranks hold identical online stats, so the merged result needs no collective)
            self.k.obs_stats_merge(self.obs_stats, self.obs_raw, self.N * self.T * self.repetitions)

    def _generation_eager(self):
        self.evaluate()
        self.rank_and_reduce()
        self.apply()

    def generation(self):
        """One full generation, device-resident; returns nothing (read .fitness_all / .update / .theta)."""
        if self._use_graph:
            if self._graph is None:
                self._capture()
            self._graph.replay()
        else:
            self._generation_eager()
        self.generation_index += 1

    def _capture(self):
        """Capture eval -> rank -> grad -> apply -> advance as one CUDA graph.  Generation / Adam counters
        live in device memory (des_state), so the same graph is replayed every generation."""
        live = [self.theta, self.adam_m, self.adam_v, self.state] + ([self.obs_stats] if self.normalize_obs else [])
        saved = [t.clone() for t in live]
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            self._generation_eager()                 # warm-up on the side stream (lazy module loading etc.)
        torch.cuda.current_stream(self.device).wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._generation_eager()
        for t, v in zip(live, saved):
            t.copy_(v)                                # capture does not execute, the warm-up did: roll it back
        self._graph = g

    # -- host-buffer entry (the reference-facing call: inputs and results live on the host) ---------------------
    def generation_host(self, obs_host, target_host, theta_out_host=None, fitness_out_host=None):
        """H2D tape -> generation -> D2H (theta, fitness).  Pinned host tensors make the copies async;
        the call returns after the results have landed."""
        self.set_tape(obs_host, target_host)
        self.generation()
        if theta_out_host is not None:
            theta_out_host.copy_(self.theta, non_blocking=True)
        if fitness_out_host is not None:
            fitness_out_host.copy_(self.fitness_all, non_blocking=True)
        if self.device.type == 'cuda':
            torch.cuda.current_stream(self.device).synchronize()

    # -- conveniences --------------------------------------------------------------------------------------
    def noiseless_fitness(self, solution=None):
        """Return of the tape episode for one flat solution (test(), natural_es.py:101-110)."""
        theta = self.theta if solution is None else torch.as_tensor(
            np.ascontiguousarray(solution, dtype=np.float32)).to(self.device)
        obs = self.obs_raw
        if self.normalize_obs:
            obs = self.k.obs_normalize(self.obs_raw, self.obs_stats)
        out = self.k.nes_eval(theta, obs, self.target, hidden=self.H, sigma=0.0, clip=self.clip, seed=self.seed,
                              generation=0, member_offset=0, n_local=1, precision='fp32')
        return float(out[0])

    def stats_state_dict(self):
        """SharedStats.state_dict (utils.py:98-101) of the device-resident statistics."""
        if not self.normalize_obs:
            z = np.zeros(self.d0, dtype=np.float32)
            return {'m': z, 'v': z.copy(), 'n': np.zeros(1, dtype=np.float32)}
        st = self.obs_stats.cpu().numpy()
        return {'m': st[:self.d0].copy(), 'v': st[self.d0:2 * self.d0].copy(), 'n': st[2 * self.d0:].copy()}

    def theta_numpy(self):
        return self.theta.detach().cpu().numpy()


class RolloutEngine(NESEngine):
    """NES generation whose fitness comes from closed-loop episodes stepped on the device (SURVEY 8f row 3): the
    reference's real workload — Evaluator.eval utils.py:116-124 runs `repetitions` episodes of the environment per
    member, every member seeing its own observations.  Environment: 'Pendulum-v0' (config.py:26-31).

    Differences from the tape engine: `evaluate` calls des_rollout_eval; the observation statistics are those of the
    states actually visited, so each rank contributes fp64 (sum, sum of squares, count) of its members' observations
    and one (2*d0+1)-double all-reduce replaces the per-worker Chan merges of natural_es.py:85-89."""

    ENVS = {'Pendulum-v0': dict(env=0, state_dim=3, action_dim=1, clip=2.0, horizon=200)}

    def __init__(self, *, task='Pendulum-v0', hidden, pop_size, theta0, sigma, learning_rate, repetitions=10,
                 horizon=None, action_noise_std=0.0, normalize_obs=True, **kw):
        if task not in self.ENVS:
            raise ValueError('closed-loop environments available on the device: %s (got %r)' % (sorted(self.ENVS), task))
        if int(hidden) not in (16, 32, 64, 96, 128):
            raise ValueError('RolloutEngine: hidden must be 16, 32, 64, 96 or 128 (des_rollout_eval keeps H/16 units per lane); '
                             'got %r' % (hidden,))
        if not (1 <= int(repetitions) <= 10):
            raise ValueError('RolloutEngine: repetitions must be in [1, 10] (one warp steps them in lockstep); got %r'
                             % (repetitions,))
        e = self.ENVS[task]
        self.env_id, self.horizon = e['env'], int(horizon or e['horizon'])
        self.action_noise_std = float(action_noise_std)
        kw.setdefault('clip', e['clip'])
        kw.pop('precision', None)
        super().__init__(state_dim=e['state_dim'], hidden=hidden, action_dim=e['action_dim'], pop_size=pop_size,
                         theta0=theta0, obs=None, target=None, sigma=sigma, learning_rate=learning_rate,
                         precision='fp32', normalize_obs=normalize_obs, repetitions=repetitions, **kw)
        if self.world > 1 and self.normalize_obs:
            self._use_graph = False          # the observation totals still travel through an NCCL all-reduce

    def _setup_inputs(self, obs, target):
        self.T = self.horizon
        self.eval_ws = None
        w = 2 * self.d0 + 1
        self.obs_totals = torch.zeros(w, dtype=torch.float64, device=self.device)
        self.roll_ws = torch.empty(max(self.n_local, 1) * w, dtype=torch.float64, device=self.device)

    def set_tape(self, obs, target):
        raise TypeError('RolloutEngine steps the environment on the device; there is no tape to set')

    def evaluate(self):
        if self.world > 1 and self.comm is None:
            self.fitness_all.zero_()
        self.obs_totals.zero_()
        if self.n_local:
            self._op('rollout_eval')(self.theta, env=self.env_id, hidden=self.H, horizon=self.horizon,
                                     repetitions=self.repetitions, sigma=self.sigma, clip=self.clip,
                                     action_noise_std=self.action_noise_std, seed=self.seed, state=self.state,
                                     member_offset=self.offset, n_local=self.n_local,
                                     obs_stats=self.obs_stats if self.normalize_obs else None,
                                     totals_out=self.obs_totals if self.normalize_obs else None, workspace=self.roll_ws,
                                     out=self.fitness_shard_out)
        self._gather_fitness()
        if self.world > 1 and self.normalize_obs:
            dist.all_reduce(self.obs_totals, group=self.pg)
        return self.fitness_all

    def _merge_obs_stats(self):
        if self.normalize_obs:
            self.k.obs_stats_merge_totals(self.obs_stats, self.obs_totals, self.d0)

    def generation_host(self, theta_out_host=None, fitness_out_host=None):
        """generation -> D2H (theta, fitness); a closed-loop generation has no per-step host input."""
        self.generation()
        if theta_out_host is not None:
            theta_out_host.copy_(self.theta, non_blocking=True)
        if fitness_out_host is not None:
            fitness_out_host.copy_(self.fitness_all, non_blocking=True)
        if self.device.type == 'cuda':
            torch.cuda.current_stream(self.device).synchronize()

    def test_returns(self, solution=None, repetitions=None):
        """Returns of `repetitions` test episodes of the unperturbed solution (test(), natural_es.py:101-110)."""
        theta = self.theta if solution is None else torch.as_tensor(
            np.ascontiguousarray(solution, dtype=np.float32)).to(self.device)
        reps = int(repetitions or self.repetitions)
        episodes = torch.empty(reps, dtype=torch.float32, device=self.device)
        self.k.rollout_eval(theta, env=self.env_id, hidden=self.H, horizon=self.horizon, repetitions=reps,
                            sigma=0.0, clip=self.clip, action_noise_std=self.action_noise_std, seed=self.seed,
                            state=self.state, member_offset=0, n_local=1, noiseless=True,
                            obs_stats=self.obs_stats if self.normalize_obs else None, episodes_out=episodes)
        return episodes.cpu().numpy().astype(np.float64)

    def noiseless_fitness(self, solution=None):
        return float(self.test_returns(solution).mean())


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

    def run(self, rows, *, generation, member_offset=0, key_member=None, obs_stats=None, stat_part=None):
        """Returns (returns[n, repetitions] fp64, environment steps taken).  Episode (i, r) resets with the key
        (generation, member_offset + i, r), or (generation, key_member, r) when key_member is given (test episodes,
        whose action noise then uses member 0 as des_rollout_eval's test episodes do)."""
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
            alive &= ~np.asarray(done, dtype=bool)
            t += 1
        return returns.reshape(n, reps), steps


class HostEnvEngine(NESEngine):
    """NES generation over environments stepped on the HOST by the user's own code (any gym-style task), with the
    population's per-step policy on the device (des_policy_act): Evaluator.eval utils.py:116-124 for every member of the
    rank's shard, `repetitions` episodes each.

    Per generation: des_nes_perturb materialises the shard's rows theta + sigma*eps once; every slot resets with its key
    (generation, global member, repetition); HostEpisodes steps until no slot is alive; fitness = mean return over the
    repetitions (utils.py:124) into the shard of fitness_all, then the fitness all-gather.  The raw observations of the
    alive slots accumulate per member on the device, are reduced in member order and, sharded, all-reduced (as
    RolloutEngine).  `steps_taken` is the number of environment steps of the generation, summed over ranks
    (natural_es.py:75).  Rank, gradient and apply are NESEngine's; the generation stays eager (the host loop is inside it).

    env_fn: a single environment with the classic gym API (probed for the dimensions); batch_env_fn(num_slots), if given,
    builds a vectorised environment implementing the batch protocol of envs.py instead of envs.GymEnvBatch."""

    HIDDEN = (16, 32, 64, 96, 128)

    def __init__(self, *, env_fn, hidden, pop_size, theta0, sigma, learning_rate, state_dim=None, action_dim=None,
                 repetitions=10, test_repetitions=None, action_noise_std=0.0, normalize_obs=True, batch_env_fn=None,
                 **kw):
        if state_dim is None or action_dim is None:
            probe = env_fn()
            state_dim, action_dim = probe.observation_space.shape[0], probe.action_space.shape[0]
        if int(hidden) not in self.HIDDEN:
            raise ValueError('HostEnvEngine: hidden must be 16, 32, 64, 96 or 128 (des_policy_act); got %r' % (hidden,))
        if not (1 <= int(state_dim) <= 32 and 1 <= int(action_dim) <= 8):
            raise ValueError('HostEnvEngine: des_policy_act takes state_dim <= 32 and action_dim <= 8; got %r, %r'
                             % (state_dim, action_dim))
        for name, r in (('repetitions', repetitions), ('test_repetitions', test_repetitions or repetitions)):
            if not (1 <= int(r) <= 16):
                raise ValueError('HostEnvEngine: %s must be in [1, 16]; got %r' % (name, r))
        self.env_fn = env_fn
        self.action_noise_std = float(action_noise_std)
        self.test_repetitions = int(test_repetitions or repetitions)
        kw.pop('precision', None)
        kw.pop('use_graph', None)
        super().__init__(state_dim=state_dim, hidden=hidden, action_dim=action_dim, pop_size=pop_size, theta0=theta0,
                         obs=None, target=None, sigma=sigma, learning_rate=learning_rate, precision='fp32',
                         normalize_obs=normalize_obs, repetitions=repetitions, **kw)
        if batch_env_fn is None:
            from .envs import GymEnvBatch
            batch_env_fn = lambda B: GymEnvBatch(env_fn, B, self.seed)      # noqa: E731
        self.batch_env_fn = batch_env_fn
        self.episodes = self._bridge(batch_env_fn(self.n_local * self.repetitions), self.n_local, self.repetitions)
        self._test_episodes = None
        self.steps_taken = 0

    def _bridge(self, batch_env, n, reps):
        return HostEpisodes(self.k, self.device, batch_env, n, reps, self.d0, self.H, self.A, self.clip,
                            self.action_noise_std, self.seed)

    def _setup_inputs(self, obs, target):
        self.T = 0                   # no fixed horizon: episodes end when the environment says so
        self.eval_ws = None
        w = 2 * self.d0 + 1
        self.rows = torch.empty((self.n_local, self.P), dtype=torch.float32, device=self.device)
        self.stat_part = torch.zeros((self.n_local, w), dtype=torch.float64, device=self.device)
        self.obs_totals = torch.zeros(w, dtype=torch.float64, device=self.device)

    def set_tape(self, obs, target):
        raise TypeError('HostEnvEngine steps its environments on the host; there is no tape to set')

    def evaluate(self):
        gen = self.generation_index
        if self.world > 1 and self.comm is None:
            self.fitness_all.zero_()
        self.obs_totals.zero_()
        steps = 0
        if self.n_local:
            self._op('nes_perturb')(self.theta, self.n_local, self.sigma, self.seed, gen, member_offset=self.offset,
                                    out=self.rows)                             # natural_es.py:28-30
            self.stat_part.zero_()
            ret, steps = self.episodes.run(self.rows, generation=gen, member_offset=self.offset,
                                           obs_stats=self.obs_stats if self.normalize_obs else None,
                                           stat_part=self.stat_part if self.normalize_obs else None)
            fit = ret.mean(axis=1)                                             # -cost, utils.py:124
            self.fitness_shard_out.copy_(torch.from_numpy(fit.astype(np.float32)))
            if self.normalize_obs:
                self.k.obs_parts_reduce(self.stat_part, self.d0, out=self.obs_totals)
        self._gather_fitness()
        total = torch.tensor([steps], dtype=torch.int64, device=self.device)
        if self.world > 1:
            if self.normalize_obs:
                dist.all_reduce(self.obs_totals, group=self.pg)
            dist.all_reduce(total, group=self.pg)
        self.steps_taken = int(total.item())
        return self.fitness_all

    def _merge_obs_stats(self):
        if self.normalize_obs:
            self.k.obs_stats_merge_totals(self.obs_stats, self.obs_totals, self.d0)

    def test_returns(self, solution=None, repetitions=None):
        """Returns of `repetitions` episodes of the unperturbed solution (test(), natural_es.py:101-110) with the current
        statistics, which they do not feed; keys (generation word, 0x40000000, repetition)."""
        from .envs import TEST_MEMBER
        theta = self.theta if solution is None else torch.as_tensor(
            np.ascontiguousarray(solution, dtype=np.float32)).to(self.device)
        reps = int(repetitions or self.test_repetitions)
        if self._test_episodes is None or self._test_episodes.reps != reps:
            self._test_episodes = self._bridge(self.batch_env_fn(reps), 1, reps)
        ret, _ = self._test_episodes.run(theta.reshape(1, -1).contiguous(), generation=self.generation_index,
                                         key_member=TEST_MEMBER,
                                         obs_stats=self.obs_stats if self.normalize_obs else None)
        return ret[0]

    def noiseless_fitness(self, solution=None):
        return float(self.test_returns(solution).mean())
