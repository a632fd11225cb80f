"""A mutation-only genetic algorithm on the fixed MLP policy (Such et al. 2017, "Deep Neuroevolution"): truncation
selection, elites and Gaussian mutation, with the surface of cma_es (GeneticAlgorithm with ask() / tell(), a Worker,
train(), test(), record() and multi_runs()).

Each generation keeps the best T members as the next parents table, the best E of them (the elites) carried over
unchanged, and fills the rest of the population with parents plus sigma * N(0, 1) noise.  The defaults are the
reference's NEAT reproduction settings (neat-config/*.txt, [DefaultReproduction]: survival_threshold = 0.2, elitism = 2):
T = ceil(0.2 N), E = 2 (at most T).  A config may set `truncation` and `elites`.

A child is fully described by (parent index, member, generation): its parent is drawn from counter stream 5 and its noise
is the member's stream-0 row, so a generation needs only the T parent rows in memory (include/des_b200.h, "genetic
algorithm").  Closed-loop configs evaluate a generation with des_rollout_eval_ga, which builds each child's weights in
shared memory; host-stepped and tape configs evaluate the rows des_ga_rows materialises.  Selection is des_ga_order, and
the next table is des_ga_rows' gather of the selected members, regenerated bit for bit as they were evaluated.

One process, one GPU: mirrored sampling and a process group of several ranks are refused.

Sweeps (train_sweep, multi_runs(batched=True)): R runs of configs that differ in seed, sigma, action noise, start point,
truncation and elites train as one batch, every run's generation one launch (des_rollout_eval_ga_sweep closed-loop, one
des_policy_act_sweep per step host-stepped), its selection one des_ga_order_runs and its next tables one
des_ga_rows_sweep gather.  Run r is train(configs[r]), bit for bit."""
from __future__ import annotations

import copy
import logging
import os
import pickle
import time

import numpy as np
import torch
import torch.distributed as dist

from . import fitness
from .cma_es import SweepWorker as _CMASweepWorker
from .engine import RankGroup, kernels_and_device
from .utils import logger

ELITISM = 2                   # neat-config/*.txt [DefaultReproduction] elitism


def default_truncation(pop_size):
    """ceil(0.2 N): neat-config/*.txt [DefaultReproduction] survival_threshold = 0.2, in integers."""
    return -(-int(pop_size) // 5)


def selection_sizes(pop_size, truncation=None, elites=None):
    """(N, T, E) with the defaults filled in; ValueError unless 2 <= N, 1 <= T <= N and 0 <= E <= T."""
    N = int(pop_size)
    if N < 2:
        raise ValueError('genetic: pop_size %d < 2: a generation needs a parent and a child' % N)
    T = default_truncation(N) if truncation is None else int(truncation)
    if not 1 <= T <= N:
        raise ValueError('genetic: truncation %d is not in [1, pop_size = %d]' % (T, N))
    E = min(ELITISM, T) if elites is None else int(elites)
    if not 0 <= E <= T:
        raise ValueError('genetic: elites %d is not in [0, truncation = %d]' % (E, T))
    return N, T, E


def _one_process(who):
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        raise ValueError('%s: the genetic algorithm trains in one process; the process group has world size %d'
                         % (who, dist.get_world_size()))


def check_config(config):
    """Raises ValueError unless genetic.train can train `config`: plain sampling, one process, and a population,
    truncation and elites in range."""
    if getattr(config, 'mirrored', False):
        raise ValueError('genetic: mirrored sampling is an NES estimator; the genetic algorithm draws one child per member '
                         '(set config.mirrored = False)')
    _one_process('genetic')
    selection_sizes(config.pop_size, getattr(config, 'truncation', None), getattr(config, 'elites', None))


class GeneticAlgorithm:
    """The parents table on the device and its generation counter.  ask() returns the generation's N rows (des_ga_rows),
    tell(fitness) selects the T best (des_ga_order) and gathers their weights into the next table.  `parents` is the
    current table [T_g, P] (one row, x0, before the first tell), `best` its row 0 and `order` the last selection.

    `kernels` (default: distributedes_b200.ops) exists so the host logic can run on CPU in the test-suite with an
    oracle-backed stand-in; the product never runs without the CUDA library."""

    def __init__(self, x0, sigma, popsize, truncation=None, elites=None, seed=0, device=None, kernels=None):
        _one_process('GeneticAlgorithm')
        self.kn, self.device = kernels_and_device(kernels, device)
        self.N, self.T, self.E = selection_sizes(popsize, truncation, elites)
        self.sigma, self.seed = float(sigma), int(seed)
        self.parents = torch.as_tensor(np.asarray(x0, dtype=np.float32).reshape(1, -1)).to(self.device).contiguous()
        self.P = int(self.parents.shape[1])
        self._spare = torch.empty((self.T, self.P), dtype=torch.float32, device=self.device)   # the next table
        self.gen = 0
        self.order = None

    @property
    def n_elites(self):
        """E_g = min(E, T_g): generation 0's table has one row."""
        return min(self.E, int(self.parents.shape[0]))

    @property
    def best(self):
        """Row 0 of the table: the best member of the last generation told (x0 before the first tell)."""
        return self.parents[0]

    def ask(self, out=None):
        """[N, P] fp32: the weights of the generation's members 0 .. N-1 (des_ga_rows)."""
        return self.kn.ga_rows(self.parents, self.n_elites, sigma=self.sigma, seed=self.seed, generation=self.gen,
                               member_offset=0, n_local=self.N, out=out)

    def tell(self, fitness, novelty=None, reward_weight=1.0):
        """Selects the T best of fitness [N] (higher is better; ties to the lower index, NaN last) and makes their
        weights, regenerated, the next table.  Returns the order [T] (int32, best first).  With novelty [N] the T first
        are those of the smallest keys fmaf(w, rank(-fitness), (1 - w) * rank(-novelty)) instead (des_ns_ga_order, w =
        reward_weight; at w = 1 the order is the fitness's, bit for bit), and the elites are the first E of them."""
        f = torch.as_tensor(fitness).to(device=self.device, dtype=torch.float32).reshape(-1).contiguous()
        if f.numel() != self.N:
            raise ValueError('tell() needs the fitness of all %d members (got %d)' % (self.N, f.numel()))
        if novelty is None:
            self.order = self.kn.ga_order(f, self.T)
        else:
            nov = torch.as_tensor(novelty).to(device=self.device, dtype=torch.float32).reshape(-1).contiguous()
            if nov.numel() != self.N:
                raise ValueError('tell() needs the novelty of all %d members (got %d)' % (self.N, nov.numel()))
            self.order = self.kn.ns_ga_order(f, nov, float(reward_weight), self.T)
        nxt = self.kn.ga_rows(self.parents, self.n_elites, sigma=self.sigma, seed=self.seed, generation=self.gen,
                              members=self.order, out=self._spare)
        self._spare = self.parents if self.parents.shape[0] == self.T else torch.empty_like(nxt)
        self.parents = nxt
        self.gen += 1
        return self.order


class Worker:
    """Evaluates a generation through the fitness source its config describes (fitness.from_config): closed-loop
    members through des_rollout_eval_ga when `fused` (the default), otherwise the rows of GeneticAlgorithm.ask() through
    the source's solutions(), as host-stepped and tape sources always do.  Holds the statistics `obs_stats`, and counts
    its test() calls in tests_run, the generation word of the next test episodes, as cma_es.Worker does."""

    def __init__(self, config, device=None, kernels=None, fused=True):
        check_config(config)
        self.config = config
        self.kn, self.device = kernels_and_device(kernels, device)
        closed = bool(getattr(config, 'closed_loop', False))
        self.source = fitness.from_config(config, self.kn, self.device, sigma=config.sigma if closed else None)
        self.fused = bool(fused) and closed
        self.group = RankGroup(None)
        self.obs_stats = self.source.obs_stats
        self.tests_run = 0
        self.fitness = self.rows = None

    def run(self, ga, bc_out=None):
        """fitness [N] fp32 (mean return, higher is better) of generation ga.gen's members; with bc_out [N, d0], the same
        evaluation also writes their behaviours (the fused closed-loop kernel, or a host-stepped source's episodes)."""
        if self.fitness is None or self.fitness.numel() != ga.N:
            self.fitness = torch.zeros(ga.N, dtype=torch.float32, device=self.device)
        bc = {} if bc_out is None else dict(bc_out=bc_out)
        if self.fused:
            self.source.ga_members(ga.parents, ga.n_elites, ga.gen, 0, ga.N, self.fitness, **bc)
        else:
            self.rows = ga.ask(out=self.rows)
            self.source.solutions(self.rows, offset=0, generation=ga.gen, out=self.fitness, **bc)
        return self.fitness

    def steps(self, N):
        """Environment steps of the last run()."""
        return self.source.steps(N, self.group)

    def test_returns(self, solution, repetitions, bc_out=None):
        """Returns of `repetitions` noiseless episodes of one solution with the current statistics; the k-th call
        (k = 0 first) resets its episodes from the test stream with generation word k.  With bc_out [1, d0], the same
        episodes also write the solution's behaviour."""
        bc = {} if bc_out is None else dict(bc_out=bc_out)
        ret = self.source.test_returns(solution, int(repetitions), self.tests_run, **bc)
        self.tests_run += 1
        return ret

    def record_test_episodes(self, solution, repetitions=None):
        """fitness.Trajectories [repetitions, horizon, ...] of the test episodes the next test_returns(solution,
        repetitions) runs: its returns are that call's.  Closed-loop configs only.  Advances nothing."""
        if not isinstance(self.source, fitness.DeviceRollouts):
            raise TypeError('%s: episodes are recorded on the device\'s closed-loop environments only (DeviceRollouts)'
                            % type(self.source).__name__)
        sol = _row(solution, self.device).reshape(-1)
        reps = repetitions or self.config.test_repetitions
        return self.source.record(sol, repetitions=int(reps), noiseless=True, generation=self.tests_run).episode(0)

    def merge_obs_stats(self, N):
        """The statistics of the last run()'s observations merged into [m|v|n]."""
        self.source.share_totals(self.group)
        self.source.merge(N)


def _row(solution, device):
    x = solution.detach().cpu() if isinstance(solution, torch.Tensor) else solution
    return torch.as_tensor(np.asarray(x, dtype=np.float32)).reshape(1, -1).to(device)


def build(config, *, kernels=None, device=None, fused=True):
    """The (Worker, GeneticAlgorithm) pair of train(config): the config's start point, sigma, population, seed and its
    optional `truncation` and `elites`."""
    worker = Worker(config, device=device, kernels=kernels, fused=fused)
    ga = GeneticAlgorithm(config.initial_weight, config.sigma, config.pop_size, truncation=getattr(config, 'truncation', None),
                          elites=getattr(config, 'elites', None), seed=config.seed, device=worker.device,
                          kernels=worker.kn)
    return worker, ga


def train(config, worker=None, ga=None):
    """Trains `config` with the genetic algorithm; returns [training_rewards, training_steps, training_timestamps] as
    cma_es.train does.  First the start point is tested.  Then each generation is evaluated, its environment steps
    counted, the next table built, its row 0 tested with test_repetitions noiseless episodes under the current statistics,
    and the generation's observation statistics merged, until max_steps or max_generations."""
    check_config(config)
    if worker is None or ga is None:
        worker, ga = build(config)
    total_steps = 0
    initial_time = time.time()
    training_rewards, training_steps, training_timestamps = [], [], []
    test_mean, test_ste = test(config, config.initial_weight, None, worker=worker)
    logger.info('total steps %d, %f(%f)' % (total_steps, test_mean, test_ste))
    training_rewards.append(test_mean)
    training_steps.append(0)
    training_timestamps.append(0)
    generation = 0
    while True:
        f = worker.run(ga)
        total_steps += worker.steps(ga.N)
        best = float(f.max())
        ga.tell(f)
        elapsed_time = time.time() - initial_time
        test_mean, test_ste = test(config, ga.best, None, worker=worker)
        logger.info('total steps %d, test %f(%f), best %f, elapsed time %f'
                    % (total_steps, test_mean, test_ste, best, elapsed_time))
        training_rewards.append(test_mean)
        training_steps.append(total_steps)
        training_timestamps.append(elapsed_time)
        worker.merge_obs_stats(ga.N)
        generation += 1
        if config.max_steps and total_steps > config.max_steps:
            break
        if getattr(config, 'max_generations', 0) and generation >= config.max_generations:
            break
    return [training_rewards, training_steps, training_timestamps]


def test(config, solution, stats, worker=None):
    """The mean and the std / repetitions (cma_es.test's formula) of `test_repetitions` noiseless episodes of one
    solution with the worker's current statistics (`stats`, if given, replaces them first)."""
    worker = worker if worker is not None else Worker(config)
    if stats is not None and worker.obs_stats is not None:
        worker.obs_stats.copy_(torch.as_tensor(np.asarray(stats, dtype=np.float32)))
    rewards = worker.test_returns(_row(solution, worker.device), config.test_repetitions)
    return np.mean(rewards), np.std(rewards) / config.repetitions


def record(config, solution, stats, worker=None):
    """test() recorded: fitness.Trajectories [test_repetitions, horizon, ...] of the test episodes whose mean
    test(config, solution, stats, worker) reports.  Closed-loop device configs only.  Advances nothing."""
    if not getattr(config, 'closed_loop', False):
        raise ValueError('genetic.record: episodes are recorded on the device\'s closed-loop environments only '
                         '(ClosedLoopPendulumConfig); a host-stepped environment\'s own code sees every step, and a tape '
                         'has no episodes')
    worker = worker if worker is not None else Worker(config)
    if stats is not None and worker.obs_stats is not None:
        worker.obs_stats.copy_(torch.as_tensor(np.asarray(stats, dtype=np.float32)))
    return worker.record_test_episodes(solution, config.test_repetitions)


def multi_runs(config, runs=10, log_dir='log', data_dir='data', kernels=None, device=None, batched=False):
    """`runs` train() runs one after the other, run r with seed config.seed + r, with the log file and the pickle of
    [[rewards, steps, timestamps], ...] of cma_es.multi_runs (data/<tag>-stats-<task>.bin, rewritten after every run).
    batched=True trains them together through train_sweep and writes the same files once: the rewards and steps are
    those of batched=False, bit for bit; the timestamps come from the sweep's one clock.  `kernels` is then a stand-in
    for ops_runs."""
    check_config(config)
    configs = []
    for run in range(runs):
        c = copy.copy(config)
        c.seed = config.seed + run
        configs.append(c)
    if batched:
        check_sweep_configs(configs)
    os.makedirs(log_dir, exist_ok=True)
    os.makedirs(data_dir, exist_ok=True)
    fh = logging.FileHandler(os.path.join(log_dir, '%s-%s.txt' % (config.tag, config.task)))
    fh.setLevel(logging.DEBUG)
    logger.addHandler(fh)
    stats = []
    path = os.path.join(data_dir, '%s-stats-%s.bin' % (config.tag, config.task))
    try:
        if batched:
            logger.info('Runs 0-%d, batched' % (runs - 1))
            stats = train_sweep(configs, *build_sweep(configs, kernels=kernels, device=device))
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
        for run in range(0 if batched else runs):
            c = configs[run]
            logger.info('Run %d' % run)
            stats.append(train(c, *build(c, kernels=kernels, device=device)))
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
    finally:
        logger.removeHandler(fh)
        fh.close()
    return stats


# ---- sweeps: R genetic-algorithm runs of different configs trained together on one GPU ----------------------------------
# The fields every config of a GA sweep shares are those of a CMA-ES sweep (cma_es.SWEEP_SHARED, SWEEP_HOST_SHARED).
# seed, sigma, action_noise_std, initial_weight, truncation and elites may differ, and host-stepped configs may have their
# own env_fn and batch_env_fn; learning_rate and weight_decay are not read.
MAX_SWEEP_POP = 2048      # the counting rank of des_ga_order_runs (larger runs are DES_ERR_UNSUPPORTED)


def check_sweep_configs(configs):
    """Raises ValueError unless train_sweep can train `configs` as one sweep: all closed-loop or all host-stepped
    configs of 2 .. 2048 members with plain sampling, in one process, each with a truncation and elites in range, that
    agree on every field of cma_es.SWEEP_SHARED (closed-loop) or cma_es.SWEEP_HOST_SHARED (host-stepped).  The first field
    that differs is named."""
    from .cma_es import SWEEP_HOST_SHARED, SWEEP_SHARED
    from .natural_es import _field, _host_sweep
    if not len(configs):
        raise ValueError('genetic.train_sweep: no configs')
    host = _host_sweep(configs)
    for i, c in enumerate(configs):
        if not host and not getattr(c, 'closed_loop', False):
            raise ValueError('genetic.train_sweep: configs[%d] is a tape config; tape configs are not batched over runs '
                             '(closed-loop ClosedLoopPendulumConfig or host-stepped HostEnvConfig only); use train()' % i)
        if getattr(c, 'mirrored', False):
            raise ValueError('genetic.train_sweep: configs[%d] asks for mirrored sampling, an NES estimator; the genetic '
                             'algorithm draws one child per member (set config.mirrored = False)' % i)
        if int(c.pop_size) > MAX_SWEEP_POP:
            raise ValueError('genetic.train_sweep: pop_size %d > %d: the runs of a sweep are ordered by the counting rank '
                             'of des_ga_order_runs, which takes up to %d members (DES_ERR_UNSUPPORTED); use train()'
                             % (c.pop_size, MAX_SWEEP_POP, MAX_SWEEP_POP))
        try:
            selection_sizes(c.pop_size, getattr(c, 'truncation', None), getattr(c, 'elites', None))
        except ValueError as e:
            raise ValueError('genetic.train_sweep: configs[%d]: %s' % (i, e)) from None
    _one_process('genetic.train_sweep')
    for i, c in enumerate(configs[1:], 1):
        for name in SWEEP_HOST_SHARED if host else SWEEP_SHARED:
            a, b = _field(configs[0], name), _field(c, name)
            if a != b:
                raise ValueError('genetic.train_sweep: configs differ in %s (%r in configs[0], %r in configs[%d]); the '
                                 'runs of a GA sweep may differ only in seed, sigma, action_noise_std, initial_weight, '
                                 'truncation and elites%s' % (name, a, b, i, ' (and, host-stepped, their own env_fn and '
                                                              'batch_env_fn)' if host else ''))


class GASweep:
    """R genetic algorithms trained as one batch on one GPU (train_sweep): strategy r is the GeneticAlgorithm of
    train(configs[r]) (x0, sigma, N, T_r, E_r, its seed), and its tables stay bit-equal to that run's.  Every run's table
    lives in one buffer [R, table_rows, P] (table_rows = max_r T_r), double-buffered; the counts of every run are the
    device table `ga` (ops_runs.ga_table), and the seeds and sigmas the rows of the sweep table `hp`.  parents[r] is run
    r's table [T_g,r, P] (a view), best[r] its row 0, order[r] its last selection [T_r] and gens[r] its generation
    counter, as GeneticAlgorithm's parents, best, order and gen.

    `running` [R] says which runs still train (train_sweep clears a run's entry where its train() would stop): stopped
    runs are neither selected nor gathered, and stop(r) detaches their table and order from the stacked buffers, frozen
    as they were at the stop."""

    def __init__(self, x0s, sigmas, popsize, truncations, elites, hp, device=None, kernels=None):
        from . import ops_runs
        _one_process('GASweep')
        self.kn, self.device = kernels_and_device(ops_runs if kernels is None else kernels, device)
        self.hp, self.R = hp, len(x0s)
        sizes = [selection_sizes(popsize, t, e) for t, e in zip(truncations, elites)]
        self.N = sizes[0][0]
        self.T = np.asarray([s[1] for s in sizes], dtype=np.int64)
        self.E = np.asarray([s[2] for s in sizes], dtype=np.int64)
        self.sigmas = [float(s) for s in sigmas]
        x0 = np.stack([np.asarray(x, dtype=np.float32).reshape(-1) for x in x0s])
        self.P, self.rows = int(x0.shape[1]), int(self.T.max())
        self.tables = torch.zeros((self.R, self.rows, self.P), dtype=torch.float32, device=self.device)
        self.tables[:, 0] = torch.from_numpy(x0).to(self.device)
        self._spare = torch.zeros_like(self.tables)
        self._order = torch.full((self.R, self.rows), -1, dtype=torch.int32, device=self.device)
        self.n_parents = np.ones(self.R, dtype=np.int64)
        self.gens = np.zeros(self.R, dtype=np.int64)
        self.gen = 0
        self.running = np.ones(self.R, dtype=bool)
        self._frozen = {}           # r -> (table, order) of a stopped run
        self.ga = self._ga_table()

    def _ga_table(self):
        return self.kn.ga_table(self.n_parents, self.n_elites, self.T, self.rows, self.device)

    @property
    def n_elites(self):
        """[R] E_g = min(E_r, T_g) of every run's current table."""
        return np.minimum(self.E, self.n_parents)

    @property
    def parents(self):
        """Run r's current table [T_g, P]: a view of the stacked buffer, or the frozen table of a stopped run."""
        return [self._frozen[r][0] if r in self._frozen else self.tables[r, :int(self.n_parents[r])]
                for r in range(self.R)]

    @property
    def best(self):
        """Row 0 of every run's table: its best member of the last generation told (x0 before the first tell)."""
        return [t[0] for t in self.parents]

    @property
    def order(self):
        """Run r's last selection [T_r] int32, best first (None before the first tell)."""
        if self.gen == 0:
            return [None] * self.R
        return [self._frozen[r][1] if r in self._frozen else self._order[r, :int(self.T[r])] for r in range(self.R)]

    def ask(self, out=None):
        """[R * N, P] fp32: run r's rows r*N .. are GeneticAlgorithm.ask() of run r (a running run's; a stopped run's
        rows are stale), from one des_ga_rows_sweep."""
        return self.kn.ga_rows_sweep(self.tables, self.ga, self.hp, generation=self.gen, run_size=self.N, out=out)

    def tell(self, fitness):
        """GeneticAlgorithm.tell() of every running run with its row of fitness [R, N]: one des_ga_order_runs and one
        des_ga_rows_sweep gather into the spare buffer, which becomes the current one.  Returns the order [R, table_rows]
        (-1 past each run's T_r)."""
        f = torch.as_tensor(fitness).to(device=self.device, dtype=torch.float32).contiguous()
        if tuple(f.shape) != (self.R, self.N):
            raise ValueError('tell() needs the fitness [R, N] = [%d, %d] of every member (got %r)'
                             % (self.R, self.N, tuple(f.shape)))
        self.kn.ga_order_runs(f, self.ga, self.rows, out=self._order)
        members = self._order
        stopped = np.flatnonzero(~self.running)
        if len(stopped):
            members = self._order.clone()
            members[torch.as_tensor(stopped, device=self.device)] = -1          # not gathered again
        self.kn.ga_rows_sweep(self.tables, self.ga, self.hp, generation=self.gen, run_size=self.N, members=members,
                              out=self._spare)
        self.tables, self._spare = self._spare, self.tables
        live = self.running.copy()
        self.n_parents[live] = self.T[live]
        self.gens[live] += 1
        self.gen += 1
        self.ga = self._ga_table()
        return self._order

    def stop(self, r):
        """Run r trains no more: its table and order leave the stacked buffers, frozen as they are."""
        order = self.order[r]
        self._frozen[r] = (self.parents[r].clone(), None if order is None else order.clone())
        self.running[r] = False


class SweepWorker(_CMASweepWorker):
    """Worker for every run of a sweep: evaluates each run's generation through one sweep source under its row of the
    table `hp` (seed, sigma and action noise) — closed-loop through fitness.DeviceSweep.ga_members (des_rollout_eval_ga_sweep,
    each member built on the device), host-stepped through fitness.HostSweep.solutions on GASweep.ask()'s rows.  Holds
    each run's statistics obs_stats and observation totals obs_totals [R, 2*d0+1], counts its test calls in tests_run as
    Worker does, and records a run's test episodes (record_test_episodes(solution, run)): cma_es.SweepWorker's."""

    def __init__(self, configs, device=None, kernels=None):
        super().__init__(configs, device=device, kernels=kernels)
        self.rows = None

    def run(self, ga):
        """fitness [R, N] fp32 (mean return, higher is better) of generation ga.gen of every run."""
        if self.fitness is None or tuple(self.fitness.shape) != (self.R, ga.N):
            self.fitness = torch.zeros((self.R, ga.N), dtype=torch.float32, device=self.device)
        if self.host:
            self.rows = ga.ask(out=self.rows)
            self.source.solutions(self.rows, self.hp, generation=ga.gen, running=ga.running, out=self.fitness)
        else:
            self.source.ga_members(ga.tables, ga.ga, self.hp, generation=ga.gen, out=self.fitness)
        return self.fitness


def build_sweep(configs, *, kernels=None, device=None):
    """The (SweepWorker, GASweep) pair of train_sweep(configs): run r has configs[r]'s seed, sigma, action noise, x0,
    truncation and elites and, host-stepped, its own environments."""
    check_sweep_configs(configs)
    worker = SweepWorker(configs, device=device, kernels=kernels)
    ga = GASweep([x.initial_weight for x in configs], [x.sigma for x in configs], configs[0].pop_size,
                 [getattr(x, 'truncation', None) for x in configs], [getattr(x, 'elites', None) for x in configs],
                 worker.hp, device=worker.device, kernels=worker.kn)
    return worker, ga


def train_sweep(configs, worker=None, ga=None):
    """train(configs[r]) for every r, trained together on one GPU: one [training_rewards, training_steps,
    training_timestamps] triple per config, whose rewards and steps are those of train(configs[r]), bit for bit (and so
    are each run's final table ga.parents[r], order ga.order[r] and statistics worker.obs_stats[r]).  The runs share one
    clock.  The configs may differ only in seed, sigma, action_noise_std, initial_weight, truncation and elites
    (check_sweep_configs); host-stepped ones also in env_fn and batch_env_fn.  Closed-loop runs all take the same steps and
    stop together; host-stepped runs count their own steps and each stops where its train() would, its environments
    never reset or stepped again and its statistics kept as they were."""
    check_sweep_configs(configs)
    if worker is None or ga is None:
        worker, ga = build_sweep(configs)
    c, R, N = configs[0], len(configs), ga.N
    out = [[[], [], []] for _ in range(R)]
    total_steps = np.zeros(R, dtype=np.int64)
    initial_time = time.time()

    def test_rows():
        return torch.stack([b.reshape(-1) for b in ga.best]).to(worker.device).contiguous()
    returns = worker.test_returns(test_rows(), c.test_repetitions, ga.running)              # test x0
    for r in range(R):
        for log, value in zip(out[r], (np.mean(returns[r]), 0, 0)):
            log.append(value)
    logger.info('total steps 0, mean over %d runs %f' % (R, float(np.mean([o[0][-1] for o in out]))))
    generation = 0
    while True:
        live = np.flatnonzero(ga.running)
        f = worker.run(ga)
        total_steps[live] += worker.steps(N)[live]
        best = f.max(dim=1).values.cpu().numpy()
        ga.tell(f)
        elapsed_time = time.time() - initial_time
        returns = worker.test_returns(test_rows(), c.test_repetitions, ga.running)         # row 0 of every table
        for r in live:
            for log, value in zip(out[r], (np.mean(returns[r]), int(total_steps[r]), elapsed_time)):
                log.append(value)
        logger.info('%d runs running, total steps %s, mean test %f, best %f, elapsed time %f'
                    % (len(live), total_steps[live].tolist(), float(np.mean([out[r][0][-1] for r in live])),
                       float(best[live].max()), elapsed_time))
        worker.merge_obs_stats(ga.running)
        generation += 1
        for r in live:                                                  # where train() breaks
            if (c.max_steps and total_steps[r] > c.max_steps) or \
                    (getattr(c, 'max_generations', 0) and generation >= c.max_generations):
                ga.stop(r)
        if not ga.running.any():
            break
    return out
