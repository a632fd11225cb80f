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
from .fitness import HostSweep


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
    def evaluate(self, bc_out=None):
        """Evaluates the generation's members; bc_out [n_local, d0], when given, also receives their behaviours from the
        same episodes (closed-loop and host-stepped sources; novelty.py)."""
        bc = {} if bc_out is None else dict(bc_out=bc_out)
        self.source.members(self.theta, state=self.state, generation=self.generation_index, offset=self.offset,
                            n_local=self.n_local, out=self.fitness_shard_out, **bc)
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

    def rank_and_reduce(self, shaped=None):
        """The shard's partial sum of shaped fitness x noise, all-reduced.  `shaped` [n_local], when given, replaces the
        centered ranks of the fitness (novelty search's blend, novelty.py)."""
        if shaped is None:
            self.k.centered_rank(self.fitness_all, self.offset, self.n_local, workspace=self.rank_ws, out=self.shaped)
            shaped = self.shaped
        grad = self.k.nes_grad_partial_mirrored if self.mirrored else self.k.nes_grad_partial
        grad(shaped, self.P, seed=self.seed, state=self.state, member_offset=self.offset, workspace=self.grad_ws,
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
    def test_returns(self, solution=None, repetitions=None, bc_out=None):
        """Returns of `repetitions` noiseless episodes of `solution` (None = theta) with the current statistics; bc_out
        [1, d0], when given, also receives the solution's behaviour from the same episodes (novelty.py)."""
        theta = self.theta if solution is None else torch.as_tensor(
            np.ascontiguousarray(solution, dtype=np.float32)).to(self.device)
        bc = {} if bc_out is None else dict(bc_out=bc_out)
        # the generation word of the test episodes: device rollouts read it from des_state, host episodes need it on
        # the host (generation_index); the tape ignores it
        return self.source.test_returns(theta, int(repetitions or self.source.test_repetitions), self.generation_index,
                                        state=self.state, **bc)

    # -- recorded episodes (closed-loop sources only) -------------------------------------------------------------
    def _recorder(self):
        if not isinstance(self.source, DeviceRollouts):
            raise TypeError('%s: episodes are recorded on the device\'s closed-loop environments only (DeviceRollouts); '
                            'a host-stepped environment\'s own code sees every step, and a tape has no episodes'
                            % type(self.source).__name__)
        return self.source

    def record_test_episodes(self, repetitions=None, solution=None):
        """fitness.Trajectories [repetitions, horizon, ...] of the test episodes test_returns(solution, repetitions) runs
        now: the same launch recorded, so its returns are test_returns()'s.  Advances nothing."""
        src = self._recorder()
        theta = self.theta if solution is None else torch.as_tensor(
            np.ascontiguousarray(solution, dtype=np.float32)).to(self.device)
        return src.record(theta, repetitions=int(repetitions or src.test_repetitions), noiseless=True,
                          state=self.state).episode(0)

    def record_members(self, first, count):
        """fitness.Trajectories [count, repetitions, horizon, ...] of members [first, first + count) of the population
        as the next evaluate() runs them (mirrored pairs whole when the engine is mirrored): the returns give that
        evaluate()'s fitness of these members bit for bit.  Advances nothing; obs_totals stay as they are."""
        first, count = int(first), int(count)
        if not (0 <= first and 0 <= count and first + count <= self.N):
            raise ValueError('record_members: members [%d, %d) are not in the population of %d' % (first, first + count,
                                                                                                  self.N))
        return self._recorder().record(self.theta, state=self.state, member_offset=first, n_local=count)

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


class _RunsUpdate:
    """The update of a batch of runs after its evaluation, one launch per step for all runs: ranking, the partial sums,
    Adam and the statistics merge.  With a sweep table `hp` each run has its own seed and hyper-parameters (ops_sweep);
    without one the runs share `seed`, `sigma`, `lr` and `wd`."""

    def rank_and_reduce(self, shaped=None):
        """Every run's partial sum of shaped fitness x noise.  `shaped` [R, N], when given, replaces the centered ranks of
        the fitness (a novelty-search sweep's blend, novelty.py)."""
        if shaped is None:
            self.k.centered_rank_runs(self.fitness_all, workspace=self.rank_ws, out=self.shaped)
            shaped = self.shaped
        if self.hp is not None:
            self.k.nes_grad_partial_sweep(shaped, self.P, self.hp, state=self.state, workspace=self.grad_ws,
                                          out=self.partial)
        else:
            self.k.nes_grad_partial_runs(shaped, self.P, seed=self.seed, state=self.state, workspace=self.grad_ws,
                                         out=self.partial)
        return self.partial

    def apply(self):
        if self.hp is not None:
            self.k.nes_apply_sweep(self.theta, self.adam_m, self.adam_v, self.partial, self.N, self.state, self.hp,
                                   beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon, update_out=self.update)
        else:
            self.k.nes_apply_runs(self.theta, self.adam_m, self.adam_v, self.partial, self.N, self.state,
                                  sigma=self.sigma, learning_rate=self.lr, weight_decay=self.wd, beta1=self.beta1,
                                  beta2=self.beta2, epsilon=self.epsilon, update_out=self.update)
        self.k.state_advance(self.state, self.beta1, self.beta2)
        if self.normalize_obs:    # natural_es.py:85-89, each run's observations into its own statistics
            self.k.obs_stats_merge_totals_runs(self.obs_stats, self.obs_totals, self.d0)

    def theta_numpy(self):
        return self.theta.detach().cpu().numpy()


class RolloutRunsEngine(_RunsUpdate):
    """R independent NES runs of `pop_size` members on the device's closed-loop Pendulum, trained together: every
    generation evaluates all runs' members in one rollout launch and ranks, reduces, applies and merges the statistics of
    all runs in one launch each, so the launches per generation do not depend on R.

    Run r's member i is the global member r*pop_size + i of the one seed (ops_runs), so run 0 is RolloutEngine's run, bit
    for bit, and runs 1..R-1 are further independent streams of the same seed, not the runs of seeds 1..R-1.  Each run has
    its own theta [R, P], fp64 Adam moments, fitness [R, N] and normaliser statistics [R, 2*d0+1]; all runs share the
    des_state (generation word, Adam's t and beta^t), the hyper-parameters and, unless theta0 is [R, P], the start point.
    `kernels` is the module of device ops (default: distributedes_b200.ops_runs); a stand-in runs the host logic on CPU.
    One GPU; the runs are not sharded.

    `seeds`, a sequence of R seeds, makes the batch a sweep (ops_sweep): run r is then RolloutEngine(seed=seeds[r],
    sigma=sigma[r], ...), bit for bit, and `sigma`, `learning_rate`, `weight_decay` and `action_noise_std` may each be
    a scalar or a sequence of R values.  Runs with equal seeds and hyper-parameters are identical.  Without `seeds` the
    hyper-parameters are scalars: the two contracts do not mix."""

    MAX_RUN_SIZE = 2048           # des_*_runs: a larger population fills the GPU without batching

    def __init__(self, *, task='Pendulum-v0', hidden, pop_size, runs, theta0, sigma, learning_rate, weight_decay=0.005,
                 repetitions=10, horizon=None, action_noise_std=0.0, normalize_obs=True, clip=None, seed=0, beta1=0.9,
                 beta2=0.999, epsilon=1e-8, use_graph=True, kernels=None, device=None, seeds=None):
        from . import ops_runs
        self.k, self.device = kernels_and_device(ops_runs if kernels is None else kernels, device)
        if self.k is ops_runs and self.device.type != 'cuda':
            raise RuntimeError('distributedes_b200 needs a CUDA device, got %s: there is no CPU fallback' % self.device)
        self.R, self.N, self.task = int(runs), int(pop_size), task
        if self.R < 1:
            raise ValueError('runs must be >= 1; got %r' % (runs,))
        if not 2 <= self.N <= self.MAX_RUN_SIZE:
            raise ValueError('RolloutRunsEngine: pop_size must be in [2, %d] (runs are batched up to the counting rank\'s '
                             'population; a larger one fills the GPU alone); got %d' % (self.MAX_RUN_SIZE, self.N))
        if self.R * self.N > 1 << 28:
            raise ValueError('RolloutRunsEngine: runs x pop_size = %d members, past 2^28' % (self.R * self.N))
        hyper = dict(sigma=sigma, learning_rate=learning_rate, weight_decay=weight_decay,
                     action_noise_std=action_noise_std)
        if seeds is None:
            for name, v in hyper.items():
                if np.ndim(v) > 0:
                    raise ValueError('RolloutRunsEngine: %s per run needs seeds= (a sweep); a batch of runs without '
                                     'seeds shares one seed and its hyper-parameters' % name)
            runs_hyper = [dict(hyper, seed=seed)]
        else:
            from .ops_sweep import per_run
            if np.ndim(seeds) == 0:
                raise ValueError('RolloutRunsEngine: seeds must be a sequence of one seed per run; got %r' % (seeds,))
            cols = dict({n: per_run(v, self.R, n) for n, v in hyper.items()}, seed=per_run(seeds, self.R, 'seeds'))
            runs_hyper = [{n: cols[n][r] for n in cols} for r in range(self.R)]
            for r, h in enumerate(runs_hyper):
                if not float(h['sigma']) > 0.0:
                    raise ValueError('RolloutRunsEngine: sigma must be > 0 (natural_es.py:92 divides by it); run %d has %r'
                                     % (r, h['sigma']))
        # the source describes the environment and its limits (one per run of a sweep); its kernels are never called
        srcs = [DeviceRollouts(self.k, self.device, task=task, hidden=hidden, repetitions=repetitions, horizon=horizon,
                               clip=clip, action_noise_std=h['action_noise_std'], seed=h['seed'],
                               normalize_obs=normalize_obs, sigma=float(h['sigma']), mirrored=False) for h in runs_hyper]
        src = srcs[0]
        self.d0, self.H, self.A, self.clip = src.d0, src.H, src.A, src.clip
        self.repetitions, self.test_repetitions, self.horizon = src.repetitions, src.test_repetitions, src.horizon
        self.env_id, self.normalize_obs = src.env_id, src.normalize_obs
        if seeds is None:
            self.action_noise_std, self.seed = src.action_noise_std, src.seed
            self.sigma, self.lr, self.wd = float(sigma), float(learning_rate), float(weight_decay)
            self.hp = None
        else:           # lists of R values, and the device table of the sweep ops
            self.seed, self.action_noise_std = [x.seed for x in srcs], [x.action_noise_std for x in srcs]
            self.sigma, self.lr, self.wd = ([float(h[n]) for h in runs_hyper]
                                            for n in ('sigma', 'learning_rate', 'weight_decay'))
            self.hp = self.k.run_table(self.seed, self.sigma, self.lr, self.wd, self.action_noise_std, self.device,
                                       runs=self.R)
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
        env = dict(env=self.env_id, hidden=self.H, horizon=self.horizon, clip=self.clip)
        return env if self.hp is not None else dict(env, action_noise_std=self.action_noise_std, seed=self.seed)

    def _rollout(self, bc_out=None, **kw):
        """rollout_eval_sweep with the table, or rollout_eval_runs with the shared seed and sigma; with bc_out,
        rollout_eval_bc_sweep, which needs the table."""
        if self.hp is not None:
            kw.pop('sigma')
            if bc_out is not None:
                return self.k.rollout_eval_bc_sweep(self.theta, self.hp, bc_out=bc_out, **kw, **self._env())
            return self.k.rollout_eval_sweep(self.theta, self.hp, **kw, **self._env())
        if bc_out is not None:
            raise ValueError('RolloutRunsEngine: behaviours (bc_out) are written for sweeps only (seeds=); a batch of runs '
                             'without seeds has none')
        return self.k.rollout_eval_runs(self.theta, **kw, **self._env())

    def evaluate(self, bc_out=None):
        """Every run's fitness [R, N]; bc_out [R, N, d0], when given, also receives the members' behaviours from the same
        episodes (a sweep only: rollout_eval_bc_sweep; novelty.py)."""
        self._rollout(repetitions=self.repetitions, sigma=self.sigma, state=self.state, run_size=self.N,
                      obs_stats=self.obs_stats, totals_out=self.obs_totals if self.normalize_obs else None,
                      workspace=self.roll_ws, out=self.fitness_all, bc_out=bc_out)
        return self.fitness_all

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

    def test_returns(self, repetitions=None, bc_out=None):
        """[R, repetitions] fp64 returns of noiseless test episodes of every run's theta with its own statistics, from
        one launch: run r's are RolloutEngine.test_returns of theta[r] (the same resets and generation word; in a sweep,
        under run r's seed).  bc_out [R, 1, d0], when given, also receives every run's behaviour from the same episodes
        (a sweep only)."""
        reps = int(repetitions or self.test_repetitions)
        episodes = torch.empty((self.R, 1, reps), dtype=torch.float32, device=self.device)
        self._rollout(repetitions=reps, sigma=0.0, state=self.state, run_size=1, noiseless=True, obs_stats=self.obs_stats,
                      out=self.test_fitness, episodes_out=episodes, bc_out=bc_out)
        return episodes.reshape(self.R, reps).cpu().numpy().astype(np.float64)

    def record_test_episodes(self, run, repetitions=None):
        """fitness.Trajectories [repetitions, horizon, ...] of run `run`'s test episodes as test_returns() runs them now,
        from one single-population launch on its theta and statistics: its returns are test_returns()[run].  In a
        sweep the run is RolloutEngine(seed=seeds[run]) at member offset 0; in a batch without seeds the run-batched
        launch keys run r's action noise by member r, so the recording does too.  Advances nothing."""
        r = int(run)
        if not 0 <= r < self.R:
            raise ValueError('record_test_episodes: run %r is not in [0, %d)' % (run, self.R))
        sweep = self.hp is not None
        src = DeviceRollouts(self.k, self.device, task=self.task, hidden=self.H, repetitions=self.repetitions,
                             horizon=self.horizon, clip=self.clip,
                             action_noise_std=self.action_noise_std[r] if sweep else self.action_noise_std,
                             seed=self.seed[r] if sweep else self.seed, normalize_obs=self.normalize_obs,
                             sigma=self.sigma[r] if sweep else self.sigma, mirrored=False)
        src.obs_stats = None if self.obs_stats is None else self.obs_stats[r]      # a view: the run's statistics now
        return src.record(self.theta[r], repetitions=int(repetitions or self.test_repetitions), noiseless=True,
                          state=self.state, member_offset=0 if sweep else r).episode(0)


class HostEnvSweepEngine(_RunsUpdate):
    """A sweep of R NES runs on environments stepped on the HOST (fitness.HostSweep): run r is HostEnvEngine(env_fn=
    env_fn[r], batch_env_fn=batch_env_fn[r], seed=seeds[r], sigma=sigma[r], ...), bit for bit, on one GPU.  Every
    environment step of every run is one des_policy_act_sweep, and every run's rows, ranking, partial sums, Adam and
    statistics merge are one launch each, so the launches per step and per generation do not depend on R.  The runs share
    the shapes, repetitions, clip, normaliser setting and Adam's beta and epsilon; `env_fn`, `batch_env_fn`, `sigma`,
    `learning_rate`, `weight_decay` and `action_noise_std` may each be one value or a sequence of R.  theta0 is [P] or
    [R, P].

    The surface is RolloutRunsEngine's, eager: evaluate() -> fitness_all [R, N], steps_taken [R], test_returns() ->
    [R, repetitions], rank_and_reduce(), apply(), generation(), theta [R, P].  `running` [R] (all True at first) says which
    runs the host loop serves: clear run r's entry once its training has ended, and its environments are never reset or
    stepped again; its slots enter every later launch dead, and what the engine computes for it is to be ignored."""

    MAX_RUN_SIZE = RolloutRunsEngine.MAX_RUN_SIZE

    def __init__(self, *, env_fn, hidden, pop_size, runs, theta0, seeds, sigma, learning_rate, weight_decay=0.005,
                 state_dim=None, action_dim=None, repetitions=10, test_repetitions=None, action_noise_std=0.0,
                 normalize_obs=True, batch_env_fn=None, clip=1.0, beta1=0.9, beta2=0.999, epsilon=1e-8, kernels=None,
                 device=None):
        from . import ops_runs
        from .ops_sweep import per_run
        self.k, self.device = kernels_and_device(ops_runs if kernels is None else kernels, device)
        if self.k is ops_runs and self.device.type != 'cuda':
            raise RuntimeError('distributedes_b200 needs a CUDA device, got %s: there is no CPU fallback' % self.device)
        self.R, self.N = int(runs), int(pop_size)
        if self.R < 1:
            raise ValueError('runs must be >= 1; got %r' % (runs,))
        if not 2 <= self.N <= self.MAX_RUN_SIZE:
            raise ValueError('HostEnvSweepEngine: pop_size must be in [2, %d] (runs are batched up to the counting rank\'s '
                             'population; a larger one fills the GPU alone); got %d' % (self.MAX_RUN_SIZE, self.N))
        if np.ndim(seeds) == 0:
            raise ValueError('HostEnvSweepEngine: seeds must be a sequence of one seed per run; got %r' % (seeds,))
        cols = dict(env_fn=env_fn, batch_env_fn=batch_env_fn, seed=seeds, sigma=sigma, learning_rate=learning_rate,
                    weight_decay=weight_decay, action_noise_std=action_noise_std)
        cols = {n: per_run(v, self.R, 'seeds' if n == 'seed' else n) for n, v in cols.items()}
        for r, s in enumerate(cols['sigma']):
            if not float(s) > 0.0:
                raise ValueError('HostEnvSweepEngine: sigma must be > 0 (natural_es.py:92 divides by it); run %d has %r'
                                 % (r, s))
        self.source = HostSweep(self.k, self.device, hidden=hidden, repetitions=repetitions, clip=clip,
                                normalize_obs=normalize_obs, state_dim=state_dim, action_dim=action_dim,
                                test_repetitions=test_repetitions,
                                runs=[dict(env_fn=cols['env_fn'][r], batch_env_fn=cols['batch_env_fn'][r],
                                           seed=cols['seed'][r], sigma=float(cols['sigma'][r]),
                                           action_noise_std=cols['action_noise_std'][r]) for r in range(self.R)])
        src = self.source
        self.d0, self.H, self.A, self.clip = src.d0, src.H, src.A, src.clip
        self.repetitions, self.test_repetitions, self.normalize_obs = src.repetitions, src.test_repetitions, src.normalize_obs
        self.seed = [x.seed for x in src.runs]
        self.action_noise_std = [x.action_noise_std for x in src.runs]
        self.sigma, self.lr, self.wd = ([float(v) for v in cols[n]] for n in ('sigma', 'learning_rate', 'weight_decay'))
        self.hp = self.k.run_table(self.seed, self.sigma, self.lr, self.wd, self.action_noise_std, self.device,
                                   runs=self.R)
        self.beta1, self.beta2, self.epsilon = float(beta1), float(beta2), float(epsilon)
        self.P = self.k.param_count(self.d0, self.H, self.A)
        theta0 = np.ascontiguousarray(theta0, dtype=np.float32)
        if theta0.size == self.P:
            theta0 = np.tile(theta0.reshape(1, -1), (self.R, 1))
        elif theta0.size != self.R * self.P:
            raise ValueError('theta0 has %d entries; the (%d,%d,%d) MLP needs %d, or %d x %d for one start point per run'
                             % (theta0.size, self.d0, self.H, self.A, self.P, self.R, self.P))
        dev, R, N, P = self.device, self.R, self.N, self.P
        self.theta = torch.from_numpy(theta0.reshape(R, P).copy()).to(dev)
        self.adam_m = torch.zeros((R, P), dtype=torch.float64, device=dev)
        self.adam_v = torch.zeros((R, P), dtype=torch.float64, device=dev)
        self.fitness_all = torch.zeros((R, N), dtype=torch.float32, device=dev)
        self.shaped = torch.zeros((R, N), dtype=torch.float32, device=dev)
        self.partial = torch.zeros((R, P), dtype=torch.float32, device=dev)
        self.update = torch.zeros((R, P), dtype=torch.float32, device=dev)
        self.obs_stats, self.obs_totals = src.obs_stats, src.obs_totals
        self.state = self.k.new_state(dev, 0)
        self.rank_ws = self.k.rank_runs_workspace(R, N, dev)
        self.grad_ws = self.k.grad_runs_workspace(R, N, P, dev)
        self.generation_index = 0
        self.steps_taken = np.zeros(R, dtype=np.int64)      # per run, the episodes' real lengths (natural_es.py:75)
        self.running = np.ones(R, dtype=bool)

    def evaluate(self, bc_out=None):
        """Every run's fitness [R, N]; bc_out [R, N, d0], when given, also receives the members' behaviours from the same
        episodes (novelty.py)."""
        bc = {} if bc_out is None else dict(bc_out=bc_out)
        self.source.members(self.theta, self.hp, generation=self.generation_index, run_size=self.N,
                            running=self.running, out=self.fitness_all, **bc)
        self.steps_taken = self.source.last_steps
        return self.fitness_all

    def generation(self):
        """One generation of every run, eager (the host loop is inside it); read .fitness_all / .theta."""
        self.evaluate()
        self.rank_and_reduce()
        self.apply()
        self.generation_index += 1

    def test_returns(self, repetitions=None, bc_out=None):
        """[R, repetitions] fp64 returns of noiseless test episodes of every running run's theta with its own statistics,
        keyed (generation_index, TEST_MEMBER, repetition): run r's are HostEnvEngine.test_returns of theta[r].  The
        runs `running` leaves out return zeros.  bc_out [R, 1, d0], when given, also receives every running run's
        behaviour from the same episodes."""
        reps = int(repetitions or self.test_repetitions)
        bc = {} if bc_out is None else dict(bc_out=bc_out)
        return self.source.test_returns(self.theta, self.hp, reps, self.generation_index, self.running, **bc)
