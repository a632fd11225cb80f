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

import os

import numpy as np
import torch
import torch.distributed as dist

from . import ops
from .fitness import DeviceRollouts, HostEpisodes, HostRollouts, Tape  # noqa: F401  (engine.HostEpisodes stays public)


def shard_bounds(N, world_size, rank):
    """Contiguous split of N members over world_size ranks; the first N % world_size ranks get one more."""
    if world_size < 1 or not (0 <= rank < world_size):
        raise ValueError('bad rank %r / world_size %r' % (rank, world_size))
    base, rem = divmod(int(N), int(world_size))
    start = rank * base + min(rank, rem)
    return start, base + (1 if rank < rem else 0)


class RankGroup:
    """This process among the ranks of `process_group`: its `world`, `rank` and `pg` (1, 0 and None when
    torch.distributed is not initialised), its shard of a population and the two collectives the trainers issue."""

    def __init__(self, process_group=None):
        self.pg = process_group
        distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(process_group) if distributed else 1
        self.rank = dist.get_rank(process_group) if distributed else 0

    def shard(self, N, pairs=False):
        """(offset, count) of this rank's members of N; with `pairs`, whole +-eps pairs (members 2p and 2p+1)."""
        if pairs:
            offset, n = shard_bounds(N // 2, self.world, self.rank)
            return 2 * offset, 2 * n
        return shard_bounds(N, self.world, self.rank)

    def sum_(self, t):
        """t summed over the ranks, in place; a single process has nothing to add."""
        if self.world > 1:
            dist.all_reduce(t, group=self.pg)
        return t

    def gather(self, part, offset, N, out=None):
        """[N, ...] on every rank from each rank's `part`, its rows [offset, offset + len(part)): the sum over the ranks
        of the zero-padded parts, which is an all-gather that allows ragged shards.  A single process returns `part` (or
        `out`).  `out`, when given, is the [N, ...] result with `part` already its slice: the gather is then in place,
        with no copy and no allocation."""
        if self.world == 1:
            return part if out is None else out
        if out is None:
            out = part.new_zeros((N,) + tuple(part.shape[1:]))
            out[offset:offset + len(part)] = part
        else:
            out[:offset].zero_()
            out[offset + len(part):].zero_()
        dist.all_reduce(out, group=self.pg)
        return out


def capture_generation(device, live, generation):
    """`generation` captured as one CUDA graph, after a warm-up run on a side stream whose effect on the `live` tensors
    (the state a generation advances) is rolled back: capture does not execute, the warm-up did."""
    saved = [t.clone() for t in live]
    s = torch.cuda.Stream(device=device)
    s.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(s):
        generation()                             # warm-up on the side stream (lazy module loading etc.)
    torch.cuda.current_stream(device).wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        generation()
    for t, v in zip(live, saved):
        t.copy_(v)
    return g


def kernels_and_device(kernels=None, device=None):
    """The device ops and the device of a trainer: `kernels` None is distributedes_b200.ops (libdes_b200.so), `device`
    None the current CUDA device.  The library has no CPU path, so it is refused a CPU device here, at construction."""
    kernels = ops if kernels is None else kernels
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if kernels is ops and device.type != 'cuda':
        raise RuntimeError('distributedes_b200 needs a CUDA device, got %s: there is no CPU fallback' % device)
    return kernels, device


class NESEngine:
    """One rank's NES generation.  `obs`, `target`, `normalize_obs` and `repetitions` build the tape source unless a
    `source` is given; the source's buffers (tape, eval workspace, statistics, host rows) and its precision read through
    the engine."""

    def __init__(self, *, state_dim, hidden, action_dim, pop_size, theta0, obs=None, target=None, sigma, learning_rate,
                 weight_decay=0.005, clip=1.0, seed=0, precision='fp32', beta1=0.9, beta2=0.999, epsilon=1e-8,
                 device=None, process_group=None, kernels=None, use_graph=False, normalize_obs=False, repetitions=1,
                 mirrored=False, source=None):
        self.k, self.device = kernels_and_device(kernels, device)
        self.group = RankGroup(process_group)
        self.world, self.rank = self.group.world, self.group.rank
        self.d0, self.H, self.A = int(state_dim), int(hidden), int(action_dim)
        self.N = int(pop_size)
        if self.N < 2:
            raise ValueError('pop_size must be >= 2 (fitness_shift divides by N-1, utils.py:146)')
        # mirrored sampling: members 2p and 2p+1 are theta +- sigma*eps_p; a shard holds whole pairs
        self.mirrored = bool(mirrored)
        if self.mirrored and self.N % 2:
            raise ValueError('mirrored sampling needs an even pop_size (members come in +-eps pairs); got %d' % self.N)
        self.offset, self.n_local = self.group.shard(self.N, pairs=self.mirrored)
        self.sigma, self.lr, self.wd, self.clip = float(sigma), float(learning_rate), float(weight_decay), float(clip)
        self.beta1, self.beta2, self.epsilon = float(beta1), float(beta2), float(epsilon)
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
        if self.world > 1 and self.k.__name__.endswith('.ops') and dev.type == 'cuda' and os.environ.get('DES_COMM', 'peer') != 'nccl':
            try:
                from .comm import PeerComm
                self.comm = PeerComm(self.N, self.P, dev, self.group)
            except RuntimeError as e:
                import warnings
                warnings.warn('distributedes_b200: peer-memory exchange unavailable (%s); using NCCL all-reduces' % e)
                self.comm = None
            # every rank must take the same path
            ok = torch.tensor([1 if self.comm is not None else 0], device=dev)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group.pg)
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
        self.source = source if source is not None else Tape(
            self.k, dev, obs, target, state_dim=self.d0, hidden=self.H, action_dim=self.A, clip=self.clip,
            repetitions=repetitions, normalize_obs=normalize_obs, sigma=self.sigma, seed=seed, precision=precision,
            mirrored=self.mirrored)
        self.generation_index = 0
        self.steps_taken = 0          # environment steps of the last evaluation, summed over ranks (natural_es.py:75)
        self._graph = None
        # the whole generation is one CUDA graph: always on a single GPU; sharded, when the exchange runs on the
        # peer-memory kernels (nothing but kernels of this library in the stream).  With NCCL collectives the generation
        # stays eager unless DES_GRAPH_NCCL=1 (capturing ProcessGroupNCCL collectives hung on the 2-GPU box in round 1).
        self._use_graph = (bool(use_graph) and self.device.type == 'cuda' and self.source.capturable(self.world)
                           and (self.world == 1 or self.comm is not None or os.environ.get('DES_GRAPH_NCCL') == '1'))

    def __getattr__(self, name):
        if name == 'source':
            raise AttributeError(name)
        return getattr(self.source, name)

    @property
    def seed(self):
        return self.source.seed

    @seed.setter
    def seed(self, value):
        self.source.seed = int(value)

    # -- the three phases around the two collectives -------------------------------------------------------
    def evaluate(self):
        self.source.members(self.theta, state=self.state, generation=self.generation_index, offset=self.offset,
                            n_local=self.n_local, out=self.fitness_shard_out)
        self._gather_fitness()
        self.source.share_totals(self.group)
        self.steps_taken = self.source.steps(self.N, self.group)
        return self.fitness_all

    @property
    def fitness_shard_out(self):
        """Where this rank's evaluation kernel writes its shard (the exchange block when peers read it from there)."""
        return self._fitness_xchg[self.offset:self.offset + self.n_local]

    def _gather_fitness(self):
        if self.comm is not None:
            self.comm.allgather_fitness(self.offset, self.n_local)     # shard -> every peer's exchange block, flag barrier
            self.fitness_all.copy_(self._fitness_xchg)                 # the stable private copy (a 4N-byte device copy)
        else:
            self.group.gather(self.fitness_shard_out, self.offset, self.N, out=self.fitness_all)

    def rank_and_reduce(self):
        self.k.centered_rank(self.fitness_all, self.offset, self.n_local, workspace=self.rank_ws, out=self.shaped)
        grad = self.k.nes_grad_partial_mirrored if self.mirrored else self.k.nes_grad_partial
        grad(self.shaped, self.P, seed=self.seed, state=self.state, member_offset=self.offset, workspace=self.grad_ws,
             out=self.partial_local if self.comm is not None else self.partial)
        if self.comm is not None:
            self.comm.allreduce_partial(self.partial_local, self.partial)   # slots over NVLink, summed in rank order
        else:
            self.group.sum_(self.partial)
        return self.partial

    def apply(self):
        self.k.nes_apply(self.theta, self.adam_m, self.adam_v, self.partial, self.N, self.state, sigma=self.sigma,
                         learning_rate=self.lr, weight_decay=self.wd, beta1=self.beta1, beta2=self.beta2,
                         epsilon=self.epsilon, update_out=self.update)
        self.k.state_advance(self.state, self.beta1, self.beta2)
        self.source.merge(self.N)         # natural_es.py:85-89: this generation's observations into the statistics

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
        self._graph = capture_generation(self.device, live, self._generation_eager)

    # -- host-buffer entry (the reference-facing call: inputs and results live on the host) ---------------------
    def set_tape(self, obs, target):
        if self.source.set_tape(obs, target):
            self._graph = None

    def generation_host(self, obs_host=None, target_host=None, theta_out_host=None, fitness_out_host=None):
        """[H2D tape ->] generation -> D2H (theta, fitness).  The tape is for engines that read one; pinned host
        tensors make the copies async; the call returns after the results have landed."""
        if obs_host is not None:
            self.set_tape(obs_host, target_host)
        self.generation()
        if theta_out_host is not None:
            theta_out_host.copy_(self.theta, non_blocking=True)
        if fitness_out_host is not None:
            fitness_out_host.copy_(self.fitness_all, non_blocking=True)
        if self.device.type == 'cuda':
            torch.cuda.current_stream(self.device).synchronize()

    # -- test episodes (test(), natural_es.py:101-110) ----------------------------------------------------------
    def test_returns(self, solution=None, repetitions=None):
        """Returns of `repetitions` noiseless episodes of `solution` (None = theta) with the current statistics."""
        theta = self.theta if solution is None else torch.as_tensor(
            np.ascontiguousarray(solution, dtype=np.float32)).to(self.device)
        # the generation word of the test episodes: device rollouts read it from des_state, host episodes need it on
        # the host (generation_index); the tape ignores it
        return self.source.test_returns(theta, int(repetitions or self.source.test_repetitions), self.generation_index,
                                        state=self.state)

    def noiseless_fitness(self, solution=None):
        return float(self.test_returns(solution).mean())

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
    """NES generation whose fitness comes from closed-loop episodes stepped on the device (fitness.DeviceRollouts):
    the reference's real workload, Evaluator.eval utils.py:116-124 with `repetitions` episodes per member.
    Environment: 'Pendulum-v0' (config.py:26-31).  Sharded with the normaliser on, the generation stays eager."""

    def __init__(self, *, task='Pendulum-v0', hidden, pop_size, theta0, sigma, learning_rate, repetitions=10,
                 horizon=None, action_noise_std=0.0, normalize_obs=True, clip=None, seed=0, mirrored=False, kernels=None,
                 device=None, **kw):
        k, dev = kernels_and_device(kernels, device)
        src = DeviceRollouts(k, dev, task=task, hidden=hidden, repetitions=repetitions, horizon=horizon, clip=clip,
                             action_noise_std=action_noise_std, seed=seed, normalize_obs=normalize_obs, sigma=float(sigma),
                             mirrored=mirrored)
        super().__init__(state_dim=src.d0, hidden=hidden, action_dim=src.A, pop_size=pop_size, theta0=theta0, sigma=sigma,
                         learning_rate=learning_rate, clip=src.clip, mirrored=mirrored, source=src, kernels=k, device=dev,
                         **kw)


class HostEnvEngine(NESEngine):
    """NES generation over environments stepped on the HOST by the user's own code (fitness.HostRollouts; env_fn is
    probed for the dimensions when they are not given).  The generation stays eager: the host loop is inside it."""

    def __init__(self, *, env_fn, hidden, pop_size, theta0, sigma, learning_rate, state_dim=None, action_dim=None,
                 repetitions=10, test_repetitions=None, action_noise_std=0.0, normalize_obs=True, batch_env_fn=None,
                 clip=1.0, seed=0, mirrored=False, kernels=None, device=None, **kw):
        k, dev = kernels_and_device(kernels, device)
        src = HostRollouts(k, dev, env_fn=env_fn, batch_env_fn=batch_env_fn, state_dim=state_dim, action_dim=action_dim,
                           hidden=hidden, repetitions=repetitions, test_repetitions=test_repetitions, clip=clip,
                           action_noise_std=action_noise_std, seed=seed, normalize_obs=normalize_obs, sigma=float(sigma),
                           mirrored=mirrored)
        super().__init__(state_dim=src.d0, hidden=hidden, action_dim=src.A, pop_size=pop_size, theta0=theta0, sigma=sigma,
                         learning_rate=learning_rate, clip=clip, mirrored=mirrored, source=src, kernels=k, device=dev,
                         **kw)


class RolloutRunsEngine:
    """R independent NES runs of `pop_size` members on the device's closed-loop Pendulum, trained together: every
    generation evaluates all runs' members in one rollout launch and ranks, reduces, applies and merges the statistics of
    all runs in one launch each, so the launches per generation do not depend on R.

    Run r's member i is the global member r*pop_size + i of the one seed (ops_runs), so run 0 is RolloutEngine's run, bit
    for bit, and runs 1..R-1 are further independent streams of the same seed, not the runs of seeds 1..R-1.  Each run has
    its own theta [R, P], fp64 Adam moments, fitness [R, N] and normaliser statistics [R, 2*d0+1]; all runs share the
    des_state (generation word, Adam's t and beta^t), the hyper-parameters and, unless theta0 is [R, P], the start point.
    `kernels` is the module of device ops (default: distributedes_b200.ops_runs); a stand-in runs the host logic on CPU.
    One GPU; the runs are not sharded."""

    MAX_RUN_SIZE = 2048           # des_*_runs: a larger population fills the GPU without batching

    def __init__(self, *, task='Pendulum-v0', hidden, pop_size, runs, theta0, sigma, learning_rate, weight_decay=0.005,
                 repetitions=10, horizon=None, action_noise_std=0.0, normalize_obs=True, clip=None, seed=0, beta1=0.9,
                 beta2=0.999, epsilon=1e-8, use_graph=True, kernels=None, device=None):
        from . import ops_runs
        self.k, self.device = kernels_and_device(ops_runs if kernels is None else kernels, device)
        if self.k is ops_runs and self.device.type != 'cuda':
            raise RuntimeError('distributedes_b200 needs a CUDA device, got %s: there is no CPU fallback' % self.device)
        self.R, self.N = int(runs), int(pop_size)
        if self.R < 1:
            raise ValueError('runs must be >= 1; got %r' % (runs,))
        if not 2 <= self.N <= self.MAX_RUN_SIZE:
            raise ValueError('RolloutRunsEngine: pop_size must be in [2, %d] (runs are batched up to the counting rank\'s '
                             'population; a larger one fills the GPU alone); got %d' % (self.MAX_RUN_SIZE, self.N))
        if self.R * self.N > 1 << 28:
            raise ValueError('RolloutRunsEngine: runs x pop_size = %d members, past 2^28' % (self.R * self.N))
        # the source describes the environment and its limits; its kernels are never called
        src = DeviceRollouts(self.k, self.device, task=task, hidden=hidden, repetitions=repetitions, horizon=horizon,
                             clip=clip, action_noise_std=action_noise_std, seed=seed, normalize_obs=normalize_obs,
                             sigma=float(sigma), mirrored=False)
        self.d0, self.H, self.A, self.clip = src.d0, src.H, src.A, src.clip
        self.repetitions, self.test_repetitions, self.horizon = src.repetitions, src.test_repetitions, src.horizon
        self.env_id, self.action_noise_std, self.seed = src.env_id, src.action_noise_std, src.seed
        self.normalize_obs = src.normalize_obs
        self.sigma, self.lr, self.wd = float(sigma), float(learning_rate), float(weight_decay)
        self.beta1, self.beta2, self.epsilon = float(beta1), float(beta2), float(epsilon)
        self.P = self.k.param_count(self.d0, self.H, self.A)
        theta0 = np.ascontiguousarray(theta0, dtype=np.float32)
        if theta0.size == self.P:
            theta0 = np.tile(theta0.reshape(1, -1), (self.R, 1))
        elif theta0.size != self.R * self.P:
            raise ValueError('theta0 has %d entries; the (%d,%d,%d) MLP needs %d, or %d x %d for one start point per run'
                             % (theta0.size, self.d0, self.H, self.A, self.P, self.R, self.P))
        dev, R, N, P, w = self.device, self.R, self.N, self.P, 2 * self.d0 + 1
        self.theta = torch.from_numpy(theta0.reshape(R, P).copy()).to(dev)
        self.adam_m = torch.zeros((R, P), dtype=torch.float64, device=dev)
        self.adam_v = torch.zeros((R, P), dtype=torch.float64, device=dev)
        self.fitness_all = torch.zeros((R, N), dtype=torch.float32, device=dev)
        self.shaped = torch.zeros((R, N), dtype=torch.float32, device=dev)
        self.partial = torch.zeros((R, P), dtype=torch.float32, device=dev)
        self.update = torch.zeros((R, P), dtype=torch.float32, device=dev)
        self.obs_stats = torch.zeros((R, w), dtype=torch.float32, device=dev) if self.normalize_obs else None
        self.obs_totals = torch.zeros((R, w), dtype=torch.float64, device=dev)
        self.roll_ws = torch.empty(R * N * w, dtype=torch.float64, device=dev)
        self.test_fitness = torch.empty((R, 1), dtype=torch.float32, device=dev)
        self.state = self.k.new_state(dev, 0)
        self.rank_ws = self.k.rank_runs_workspace(R, N, dev)
        self.grad_ws = self.k.grad_runs_workspace(R, N, P, dev)
        self.generation_index = 0
        self.steps_taken = N * self.repetitions * self.horizon      # per run (natural_es.py:75)
        self._graph = None
        self._use_graph = bool(use_graph) and dev.type == 'cuda'

    def _env(self):
        return dict(env=self.env_id, hidden=self.H, horizon=self.horizon, clip=self.clip,
                    action_noise_std=self.action_noise_std, seed=self.seed)

    def evaluate(self):
        self.k.rollout_eval_runs(self.theta, repetitions=self.repetitions, sigma=self.sigma, state=self.state,
                                 run_size=self.N, obs_stats=self.obs_stats,
                                 totals_out=self.obs_totals if self.normalize_obs else None, workspace=self.roll_ws,
                                 out=self.fitness_all, **self._env())
        return self.fitness_all

    def rank_and_reduce(self):
        self.k.centered_rank_runs(self.fitness_all, workspace=self.rank_ws, out=self.shaped)
        self.k.nes_grad_partial_runs(self.shaped, self.P, seed=self.seed, state=self.state, workspace=self.grad_ws,
                                     out=self.partial)
        return self.partial

    def apply(self):
        self.k.nes_apply_runs(self.theta, self.adam_m, self.adam_v, self.partial, self.N, self.state, sigma=self.sigma,
                              learning_rate=self.lr, weight_decay=self.wd, beta1=self.beta1, beta2=self.beta2,
                              epsilon=self.epsilon, update_out=self.update)
        self.k.state_advance(self.state, self.beta1, self.beta2)
        if self.normalize_obs:    # natural_es.py:85-89, each run's observations into its own statistics
            self.k.obs_stats_merge_totals_runs(self.obs_stats, self.obs_totals, self.d0)

    def _generation_eager(self):
        self.evaluate()
        self.rank_and_reduce()
        self.apply()

    def generation(self):
        """One generation of every run, device-resident (a replayed CUDA graph on the GPU); read .fitness_all / .theta."""
        if self._use_graph:
            if self._graph is None:
                live = [self.theta, self.adam_m, self.adam_v, self.state] + ([self.obs_stats] if self.normalize_obs else [])
                self._graph = capture_generation(self.device, live, self._generation_eager)
            self._graph.replay()
        else:
            self._generation_eager()
        self.generation_index += 1

    def test_returns(self, repetitions=None):
        """[R, repetitions] fp64 returns of noiseless test episodes of every run's theta with its own statistics, from
        one launch: run r's are RolloutEngine.test_returns of theta[r] (the same resets and generation word)."""
        reps = int(repetitions or self.test_repetitions)
        episodes = torch.empty((self.R, 1, reps), dtype=torch.float32, device=self.device)
        self.k.rollout_eval_runs(self.theta, repetitions=reps, sigma=0.0, state=self.state, run_size=1, noiseless=True,
                                 obs_stats=self.obs_stats, out=self.test_fitness, episodes_out=episodes, **self._env())
        return episodes.reshape(self.R, reps).cpu().numpy().astype(np.float64)

    def theta_numpy(self):
        return self.theta.detach().cpu().numpy()
