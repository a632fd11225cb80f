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

One process, one GPU: mirrored sampling and a process group of several ranks are refused."""
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

    def tell(self, fitness):
        """Selects the T best of fitness [N] (higher is better; ties to the lower index, NaN last) and makes their
        weights, regenerated, the next table.  Returns the order [T] (int32, best first)."""
        f = torch.as_tensor(fitness).to(device=self.device, dtype=torch.float32).reshape(-1).contiguous()
        if f.numel() != self.N:
            raise ValueError('tell() needs the fitness of all %d members (got %d)' % (self.N, f.numel()))
        self.order = self.kn.ga_order(f, self.T)
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

    def run(self, ga):
        """fitness [N] fp32 (mean return, higher is better) of generation ga.gen's members."""
        if self.fitness is None or self.fitness.numel() != ga.N:
            self.fitness = torch.zeros(ga.N, dtype=torch.float32, device=self.device)
        if self.fused:
            self.source.ga_members(ga.parents, ga.n_elites, ga.gen, 0, ga.N, self.fitness)
        else:
            self.rows = ga.ask(out=self.rows)
            self.source.solutions(self.rows, offset=0, generation=ga.gen, out=self.fitness)
        return self.fitness

    def steps(self, N):
        """Environment steps of the last run()."""
        return self.source.steps(N, self.group)

    def test_returns(self, solution, repetitions):
        """Returns of `repetitions` noiseless episodes of one solution with the current statistics; the k-th call
        (k = 0 first) resets its episodes from the test stream with generation word k."""
        ret = self.source.test_returns(solution, int(repetitions), self.tests_run)
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


def multi_runs(config, runs=10, log_dir='log', data_dir='data', kernels=None, device=None):
    """`runs` train() runs one after the other, run r with seed config.seed + r, with the log file and the pickle of
    [[rewards, steps, timestamps], ...] of cma_es.multi_runs (data/<tag>-stats-<task>.bin, rewritten after every run)."""
    check_config(config)
    os.makedirs(log_dir, exist_ok=True)
    os.makedirs(data_dir, exist_ok=True)
    fh = logging.FileHandler(os.path.join(log_dir, '%s-%s.txt' % (config.tag, config.task)))
    fh.setLevel(logging.DEBUG)
    logger.addHandler(fh)
    stats = []
    path = os.path.join(data_dir, '%s-stats-%s.bin' % (config.tag, config.task))
    try:
        for run in range(runs):
            c = copy.copy(config)
            c.seed = config.seed + run
            logger.info('Run %d' % run)
            stats.append(train(c, *build(c, kernels=kernels, device=device)))
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
    finally:
        logger.removeHandler(fh)
        fh.close()
    return stats
