"""Novelty search for NES (Conti et al. 2018, "Improving Exploration in Evolution Strategies for Deep Reinforcement
Learning via a Population of Novelty-Seeking Agents"): NS-ES, NSR-ES and NSRA-ES over the NES engine, with the surface of
natural_es (build(), train(), test()).

A member's behaviour (BC) is the raw observation its environment returns after the last step of each of its episodes,
averaged over its repetitions: d = state_dim numbers, (cos th, sin th, thdot) at the end of the episode on Pendulum.  Its
novelty is the mean distance to its k nearest behaviours in an archive (des_novelty).  Each generation shapes
fmaf(w, rank(fitness), (1 - w) * rank(novelty)) (des_ns_shape) in place of the centered ranks of the fitness: w = 0 is
NS-ES, w = 0.5 NSR-ES, and 'adaptive' is NSRA-ES, whose w starts at 1, rises by ADAPT_STEP after a test that beats the
best so far and falls by ADAPT_STEP after ADAPT_PATIENCE generations without one.  With w = 1 the generation is NES's,
bit for bit.

A meta-population of M agents (each its own engine.NESEngine: fitness source, statistics, Adam state; agent m under seed
config.seed + m) shares the archive.  Every agent's start point is tested first and its BC archived.  Each generation
picks agent m with probability proportional to the novelty of its latest BC (one des_novelty launch over the M agents),
evaluates its population (fitness and BCs from one launch), shapes, steps it, then tests it: that BC joins the archive.

Config attributes, read with defaults: ns_k (10), ns_reward_weight (0.5, or 'adaptive'), ns_agents (1).  Closed-loop and
host-stepped configs only (a tape has no episodes), plain sampling, one process.

train_sweep(configs) trains R one-agent configs as one batch on one GPU (NoveltySweep): run r is train(configs[r]), bit
for bit, and each run has its own seed, hyper-parameters, start point, archive and reward weight.  multi_runs is the
reference's driver of ten runs, sequential or batched.

train_ga(config) is novelty search for the genetic algorithm (Such et al. 2017: GA-NS, and GA-NSR / GA-NSRA with the
reward weights above), with genetic.train's loop (NoveltyGA).  The members' behaviours come from the generation's own
evaluation, and truncation selection orders fmaf(w, rank(-fitness), (1 - w) * rank(-novelty)) ascending
(des_ns_ga_order): w = 1 is genetic.train, bit for bit.  The archive takes one behaviour per generation, that of the
tested best row, and novelty is measured against the archive alone; this is this project's rule, the one train() uses,
not necessarily the paper's."""
from __future__ import annotations

import copy
import logging
import os
import pickle
import time

import numpy as np
import torch
import torch.distributed as dist

from . import genetic, natural_es
from .engine import kernels_and_device
from .model import StandardFCNet
from .utils import logger

K_DEFAULT = 10                 # nearest neighbours (Conti et al. 2018)
REWARD_WEIGHT_DEFAULT = 0.5    # NSR-ES
ADAPT_STEP = 0.05              # NSRA-ES: the change of w
ADAPT_PATIENCE = 10            # NSRA-ES: generations without a better test before w falls
MAX_K = MAX_D = 32             # des_novelty's limits
_INITIAL_CAPACITY = 64         # archive rows allocated before the first doubling


def settings(config):
    """(k, reward weight, adaptive, agents) of a config, ValueError when one is out of range."""
    k = int(getattr(config, 'ns_k', K_DEFAULT))
    w = getattr(config, 'ns_reward_weight', REWARD_WEIGHT_DEFAULT)
    M = int(getattr(config, 'ns_agents', 1))
    if not 1 <= k <= MAX_K:
        raise ValueError('novelty: ns_k %d is not in [1, %d]' % (k, MAX_K))
    if M < 1:
        raise ValueError('novelty: ns_agents must be >= 1; got %d' % M)
    adaptive = isinstance(w, str)
    if adaptive and w != 'adaptive':
        raise ValueError("novelty: ns_reward_weight must be a number in [0, 1] or 'adaptive' (NSRA-ES); got %r" % (w,))
    if not adaptive:
        w = float(w)
        if not 0.0 <= w <= 1.0:
            raise ValueError('novelty: ns_reward_weight %r is not in [0, 1]' % (w,))
    return k, w, adaptive, M


def check_config(config):
    """Raises ValueError unless novelty.train can train `config`: a closed-loop or host-stepped environment (a tape has no
    episodes, so no behaviour), plain sampling, one process, and k, d = state_dim, the agents and the reward weight in
    range."""
    if not (getattr(config, 'closed_loop', False) or getattr(config, 'host_env', False)):
        raise ValueError('novelty: a tape has no episodes and so no behaviour; novelty search needs a closed-loop '
                         '(ClosedLoopPendulumConfig) or host-stepped (HostEnvConfig) environment')
    if getattr(config, 'mirrored', False):
        raise ValueError('novelty: mirrored sampling is not supported (set config.mirrored = False)')
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        raise ValueError('novelty: novelty search trains in one process; the process group has world size %d'
                         % dist.get_world_size())
    if not 1 <= int(config.state_dim) <= MAX_D:
        raise ValueError('novelty: the behaviour has state_dim = %d entries; des_novelty takes [1, %d]'
                         % (config.state_dim, MAX_D))
    settings(config)


def _adapted(w, stall, improved):
    """NSRA-ES after a generation's test: (w, stall) -> (w, stall)."""
    if improved:
        return min(1.0, w + ADAPT_STEP), 0
    stall += 1
    if stall >= ADAPT_PATIENCE:
        return max(0.0, w - ADAPT_STEP), 0
    return w, stall


class Archive:
    """Behaviours in the order they were added: `rows` [A, d] is a view of the device buffer, whose capacity doubles
    when full."""

    def __init__(self, d, device):
        self.buffer = torch.zeros((_INITIAL_CAPACITY, int(d)), dtype=torch.float32, device=device)
        self.size = 0

    @property
    def rows(self):
        return self.buffer[:self.size]

    def add(self, row):
        if self.size == self.buffer.shape[0]:
            grown = torch.zeros((2 * self.size, self.buffer.shape[1]), dtype=torch.float32, device=self.buffer.device)
            grown[:self.size].copy_(self.buffer)
            self.buffer = grown
        self.buffer[self.size].copy_(row.reshape(-1))
        self.size += 1


class NoveltySearch:
    """The meta-population and its archive.  `agents` are the M engines, `archive` the [A, d] view of the device archive
    (capacity doubled when full), `reward_weight` the current w, `weights` the w each generation shaped with, `selected`
    the agent of each generation, `best` the best test mean so far and `best_theta` the weights that scored it.

    `kernels` (default: distributedes_b200.ops) exists so the host logic can run on CPU in the test-suite with an
    oracle-backed stand-in; the product never runs without the CUDA library."""

    def __init__(self, config, *, kernels=None, device=None):
        check_config(config)
        self.kn, self.device = kernels_and_device(kernels, device)
        self.k, w, self.adaptive, M = settings(config)
        self.reward_weight = 1.0 if self.adaptive else w
        self.agents = []
        for m in range(M):
            c = copy.copy(config)
            c.seed = config.seed + m
            theta0 = config.initial_weight if m == 0 else StandardFCNet(config.state_dim, config.action_dim,
                                                                        config.hidden_size, seed=m).get_weight()
            self.agents.append(natural_es.build_engine(c, theta0, kernels=self.kn, device=self.device))
        e = self.agents[0]
        self.d, self.N, dev = e.d0, e.N, self.device
        self.store = Archive(self.d, dev)
        self.agent_bc = torch.zeros((M, self.d), dtype=torch.float32, device=dev)     # each agent's latest behaviour
        self.bc = torch.zeros((self.N, self.d), dtype=torch.float32, device=dev)      # the members' behaviours
        self.novelty = torch.zeros(self.N, dtype=torch.float32, device=dev)
        self.shaped = torch.zeros(self.N, dtype=torch.float32, device=dev)
        self.shape_ws = self.kn.ns_shape_workspace(self.N, dev)
        self.rng = np.random.Generator(np.random.PCG64(config.seed))
        self.selected, self.weights = [], []
        self.best, self.best_theta, self.stall = -np.inf, None, 0

    @property
    def archive(self):
        return self.store.rows

    @property
    def size(self):
        return self.store.size

    @property
    def _archive(self):
        return self.store.buffer

    def _archive_add(self, row):
        self.store.add(row)

    def test_agent(self, m, repetitions):
        """natural_es.test of agent m's theta (mean, std / repetitions); the same launch writes its behaviour, which joins
        the archive.  Keeps the best test mean and its weights."""
        rewards = self.agents[m].test_returns(None, repetitions, bc_out=self.agent_bc[m:m + 1])
        self._archive_add(self.agent_bc[m])
        mean, ste = np.mean(rewards), np.std(rewards) / repetitions
        improved = bool(mean > self.best)
        if improved:
            self.best, self.best_theta = mean, self.agents[m].theta_numpy().copy()
        return mean, ste, improved

    def adapt(self, improved):
        """NSRA-ES's schedule of w after a generation's test; a fixed weight stays as it is."""
        if self.adaptive:
            self.reward_weight, self.stall = _adapted(self.reward_weight, self.stall, improved)

    def select(self):
        """The agent of the next generation, drawn with probability proportional to the novelty of its latest behaviour
        against the archive (non-finite novelty counts as 0; all zero draws uniformly).  One agent needs no draw."""
        M = len(self.agents)
        if M == 1:
            return 0
        nov = self.kn.novelty(self.agent_bc, self.archive, self.k).cpu().numpy().astype(np.float64)
        p = np.where(np.isfinite(nov), nov, 0.0)
        return int(self.rng.choice(M, p=p / p.sum() if p.sum() > 0 else None))

    def evaluate(self, m):
        """Agent m's generation: fitness (engine.fitness_all) and the members' behaviours (self.bc) from one launch."""
        return self.agents[m].evaluate(bc_out=self.bc)

    def step(self, m):
        """The members' novelty against the archive, the blend with weight w, and agent m's gradient and Adam step."""
        e = self.agents[m]
        self.kn.novelty(self.bc, self.archive, self.k, out=self.novelty)
        self.kn.ns_shape(e.fitness_all, self.novelty, self.reward_weight, workspace=self.shape_ws, out=self.shaped)
        self.weights.append(self.reward_weight)
        e.rank_and_reduce(shaped=self.shaped)
        e.apply()
        e.generation_index += 1


def build(config, *, kernels=None, device=None):
    """The NoveltySearch of train(config)."""
    return NoveltySearch(config, kernels=kernels, device=device)


def train(config, ns=None):
    """Novelty search on `config`; returns [training_rewards, training_steps, training_timestamps] with natural_es.train's
    loop, stopping rules, steps accounting and log lines.  rewards[g] is the test mean of the agent tested at the top of
    generation g: agent 0's start point at g = 0, then the agent that generation g - 1 stepped.  With one agent and
    ns_reward_weight = 1 it is natural_es.train(config), bit for bit."""
    check_config(config)
    ns = ns if ns is not None else build(config)
    reps = config.test_repetitions
    training_rewards, training_steps, training_timestamps = [], [], []
    initial_time = time.time()
    total_steps = 0
    iteration = 0
    m = 0
    while True:
        if iteration == 0:                                                     # every agent's start point
            test_mean, test_ste, _ = ns.test_agent(0, reps)
            for a in range(1, len(ns.agents)):
                ns.test_agent(a, reps)
        else:
            test_mean, test_ste, improved = ns.test_agent(m, reps)
            ns.adapt(improved)
        elapsed_time = time.time() - initial_time
        training_rewards.append(test_mean)
        training_steps.append(total_steps)
        training_timestamps.append(elapsed_time)
        logger.info('Test: total steps %d, %f(%f), elapsed time %d' % (total_steps, test_mean, test_ste, elapsed_time))

        m = ns.select()
        ns.selected.append(m)
        rewards = ns.evaluate(m)
        total_steps += ns.agents[m].steps_taken
        r_mean = float(rewards.mean())
        r_std = float(rewards.std(unbiased=False))
        logger.info('Train: iteration %d, %f(%f)' % (iteration, r_mean, r_std / np.sqrt(config.pop_size)))
        iteration += 1
        if config.max_steps and total_steps > config.max_steps:
            break
        if getattr(config, 'max_generations', 0) and iteration > config.max_generations:
            break
        ns.step(m)
    return [training_rewards, training_steps, training_timestamps]


def test(config, solution, stats, ns=None, agent=0):
    """natural_es.test: the mean and std / test_repetitions of noiseless episodes of `solution` (None = the agent's
    current weights) with agent `agent`'s statistics; without `ns`, natural_es.test's host evaluation with `stats`."""
    return natural_es.test(config, solution, stats, engine=None if ns is None else ns.agents[agent])


# ---- the genetic algorithm's novelty search: GA-NS, GA-NSR and GA-NSRA (Such et al. 2017) --------------------------------
def check_ga_config(config):
    """Raises ValueError unless train_ga can train `config`: what check_config and genetic.check_config accept, with one
    agent."""
    check_config(config)
    M = settings(config)[3]
    if M != 1:
        raise ValueError('novelty.train_ga: ns_agents = %d; the genetic algorithm evolves one population (the '
                         'meta-population of agents is an NES construction), so ns_agents must be 1' % M)
    genetic.check_config(config)


class NoveltyGA:
    """The genetic algorithm's novelty search: genetic's (Worker, GeneticAlgorithm) pair `worker`, `ga`, and an archive
    of behaviours.  Each generation's members write their behaviours from the evaluation's own launch (closed-loop:
    des_rollout_eval_ga_bc; host-stepped: the final observations of their episodes).  Their novelty against the archive
    (des_novelty) and their fitness select the next parents (des_ns_ga_order, reward weight w), and the test of the new
    best row writes the behaviour that joins the archive: one row per generation, after the start point's.  Novelty is
    measured against the archive alone, not against the current population.

    `reward_weight` is the current w, `weights` the w of each selection, `best` the best test mean so far and
    `best_theta` the weights that scored it.  `kernels` (default: distributedes_b200.ops) exists so the host logic can run
    on CPU with an oracle-backed stand-in."""

    def __init__(self, config, *, kernels=None, device=None):
        check_ga_config(config)
        self.config = config
        self.worker, self.ga = genetic.build(config, kernels=kernels, device=device)
        self.kn, self.device = self.worker.kn, self.worker.device
        self.k, w, self.adaptive, _ = settings(config)
        self.reward_weight = 1.0 if self.adaptive else w
        self.d, self.N, dev = self.worker.source.d0, self.ga.N, self.device
        self.store = Archive(self.d, dev)
        self.bc = torch.zeros((self.N, self.d), dtype=torch.float32, device=dev)       # the members' behaviours
        self.test_bc = torch.zeros((1, self.d), dtype=torch.float32, device=dev)
        self.novelty = torch.zeros(self.N, dtype=torch.float32, device=dev)
        self.weights = []
        self.best, self.best_theta, self.stall = -np.inf, None, 0

    @property
    def archive(self):
        return self.store.rows

    def test(self, solution):
        """genetic.test of one solution with the worker's statistics (mean, std / repetitions, improved); the same
        episodes write its behaviour, which joins the archive.  Keeps the best test mean and its weights."""
        c = self.config
        row = genetic._row(solution, self.device)
        rewards = self.worker.test_returns(row, c.test_repetitions, bc_out=self.test_bc)
        self.store.add(self.test_bc[0])
        mean, ste = np.mean(rewards), np.std(rewards) / c.repetitions
        improved = bool(mean > self.best)
        if improved:
            self.best, self.best_theta = mean, row.reshape(-1).cpu().numpy().copy()
        return mean, ste, improved

    def adapt(self, improved):
        """GA-NSRA's schedule of w after a generation's test (NSRA-ES's); a fixed weight stays as it is."""
        if self.adaptive:
            self.reward_weight, self.stall = _adapted(self.reward_weight, self.stall, improved)

    def evaluate(self):
        """The generation's fitness [N] (worker.run) and the members' behaviours (self.bc) from one evaluation."""
        return self.worker.run(self.ga, bc_out=self.bc)

    def select(self, fitness):
        """The members' novelty against the archive and the selection of the next parents with weight w."""
        self.kn.novelty(self.bc, self.archive, self.k, out=self.novelty)
        self.weights.append(self.reward_weight)
        return self.ga.tell(fitness, self.novelty, self.reward_weight)


def build_ga(config, *, kernels=None, device=None):
    """The NoveltyGA of train_ga(config)."""
    return NoveltyGA(config, kernels=kernels, device=device)


def train_ga(config, nsga=None):
    """The genetic algorithm's novelty search on `config`; returns [training_rewards, training_steps,
    training_timestamps] with genetic.train's loop, stopping rules, steps accounting and log lines.  ns_reward_weight 0
    is GA-NS, 0.5 (the default) GA-NSR and 'adaptive' GA-NSRA (w from 1, NSRA-ES's schedule); truncation and elites are
    genetic's.  At ns_reward_weight = 1 it is genetic.train(config), bit for bit."""
    check_ga_config(config)
    nsga = nsga if nsga is not None else build_ga(config)
    worker, ga = nsga.worker, nsga.ga
    total_steps = 0
    initial_time = time.time()
    training_rewards, training_steps, training_timestamps = [], [], []
    test_mean, test_ste, _ = nsga.test(config.initial_weight)
    logger.info('total steps %d, %f(%f)' % (total_steps, test_mean, test_ste))
    training_rewards.append(test_mean)
    training_steps.append(0)
    training_timestamps.append(0)
    generation = 0
    while True:
        f = nsga.evaluate()
        total_steps += worker.steps(ga.N)
        best = float(f.max())
        nsga.select(f)
        elapsed_time = time.time() - initial_time
        test_mean, test_ste, improved = nsga.test(ga.best)
        nsga.adapt(improved)
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


def test_ga(config, solution, stats, nsga=None):
    """genetic.test: the mean and std / repetitions of test_repetitions noiseless episodes of `solution` with the
    worker's statistics (`stats`, if given, replaces them first); without `nsga`, with a new genetic.Worker."""
    return genetic.test(config, solution, stats, worker=None if nsga is None else nsga.worker)


# ---- sweeps: R one-agent novelty searches of different configs trained together on one GPU ------------------------------
def check_sweep_configs(configs):
    """Raises ValueError unless train_sweep can train `configs` as one sweep, naming the config and the field: each
    config passes check_config and has one agent, and the list passes natural_es.check_sweep_configs (all closed-loop or
    all host-stepped, at most 2048 members each, shared fields equal) with ns_k shared too."""
    from .natural_es import SWEEP_HOST_SHARED, SWEEP_SHARED, _field, _host_sweep, check_host_sweep_config, check_runs_config
    if not len(configs):
        raise ValueError('novelty.train_sweep: no configs')
    for i, c in enumerate(configs):
        try:
            check_config(c)
        except ValueError as e:
            raise ValueError('novelty.train_sweep: configs[%d]: %s' % (i, e)) from None
        M = settings(c)[3]
        if M != 1:
            raise ValueError('novelty.train_sweep: configs[%d] has ns_agents = %d; a sweep trains one agent per run (agents '
                             'step in different generations, so each has its own Adam t, beta^t and generation word, '
                             'and the runs of a sweep share one des_state)' % (i, M))
    host = _host_sweep(configs)
    for i, c in enumerate(configs):
        try:
            (check_host_sweep_config if host else check_runs_config)(c)
        except ValueError as e:
            raise ValueError('novelty.train_sweep: configs[%d]: %s' % (i, e)) from None
    shared = (SWEEP_HOST_SHARED if host else SWEEP_SHARED) + ('ns_k',)
    for i, c in enumerate(configs[1:], 1):
        for name in shared:
            a, b = ((settings(x)[0] for x in (configs[0], c)) if name == 'ns_k' else
                    (_field(configs[0], name), _field(c, name)))
            if a != b:
                raise ValueError('novelty.train_sweep: configs differ in %s (%r in configs[0], %r in configs[%d]); the runs '
                                 'of a novelty sweep may differ only in seed, sigma, learning_rate, weight_decay, '
                                 'action_noise_std, initial_weight and ns_reward_weight%s'
                                 % (name, a, b, i, ' (and, host-stepped, their own env_fn and batch_env_fn)' if host else ''))


class NoveltySweep:
    """R one-agent novelty searches trained as one batch (train_sweep): run r is the NoveltySearch of train(configs[r]).
    `engine` is the sweep engine of natural_es.build_sweep_engine (closed-loop RolloutRunsEngine, host-stepped
    HostEnvSweepEngine); each run has its own archive [A, d] (archive(r): a view of one [R, capacity, d] buffer whose
    capacity doubles when full), reward weight (reward_weight[r], stall[r], weights[r]: the w of each generation it
    shaped with), best test mean best[r] and best_theta[r].  Every live run adds one behaviour per generation, so the live
    runs' archives have the same number of rows.

    `running` [R] says which runs still train: a host-stepped run stops where its train() would, and its archive, theta,
    Adam moments and statistics stay as they were then (theta(r), adam_m(r), adam_v(r), obs_stats(r)).  `kernels`
    (default: distributedes_b200.ops_runs) exists so the host logic can run on CPU with a stand-in."""

    def __init__(self, configs, *, kernels=None, device=None):
        check_sweep_configs(configs)
        self.engine = e = natural_es.build_sweep_engine(configs, kernels=kernels, device=device)
        self.kn, self.device, self.R, self.N, self.d = e.k, e.device, e.R, e.N, e.d0
        self.host = bool(getattr(configs[0], 'host_env', False))
        self.k = settings(configs[0])[0]
        self.adaptive = [settings(c)[2] for c in configs]
        self.reward_weight = [1.0 if a else settings(c)[1] for a, c in zip(self.adaptive, configs)]
        self.stall = [0] * self.R
        self.best, self.best_theta = [-np.inf] * self.R, [None] * self.R
        self.weights = [[] for _ in range(self.R)]
        self.running = np.ones(self.R, dtype=bool)
        R, N, d, dev = self.R, self.N, self.d, self.device
        self._archive = torch.zeros((R, _INITIAL_CAPACITY, d), dtype=torch.float32, device=dev)
        self.size = 0                                   # rows of every live run's archive
        self.sizes = np.zeros(R, dtype=np.int64)        # rows of each run's archive (a stopped run's stays)
        self.test_bc = torch.zeros((R, 1, d), dtype=torch.float32, device=dev)
        self.bc = torch.zeros((R, N, d), dtype=torch.float32, device=dev)
        self.novelty = torch.zeros((R, N), dtype=torch.float32, device=dev)
        self.shaped = torch.zeros((R, N), dtype=torch.float32, device=dev)
        self.shape_ws = self.kn.ns_shape_runs_workspace(R, N, dev)
        self.weight_table = self.kn.ns_weight_table(self.reward_weight, dev)
        self._table_weights = list(self.reward_weight)
        self._frozen = {}                               # r -> theta, Adam moments and statistics of a stopped run

    def archive(self, r):
        """Run r's archive [A_r, d]: the behaviours of its tests, in order."""
        return self._archive[r, :int(self.sizes[r])]

    def _state(self, r, name):
        if r in self._frozen:
            return self._frozen[r][name]
        t = getattr(self.engine, name)
        return None if t is None else t[r]

    def theta(self, r):
        return self._state(r, 'theta')

    def adam_m(self, r):
        return self._state(r, 'adam_m')

    def adam_v(self, r):
        return self._state(r, 'adam_v')

    def obs_stats(self, r):
        return self._state(r, 'obs_stats')

    def test(self, repetitions):
        """Every live run's test (mean, std / repetitions, improved), None for a stopped run; the same launch writes
        each run's behaviour, which joins its archive.  Keeps each run's best test mean and its weights."""
        e = self.engine
        returns = e.test_returns(repetitions, bc_out=self.test_bc)
        if self.size == self._archive.shape[1]:
            grown = torch.zeros((self.R, 2 * self.size, self.d), dtype=torch.float32, device=self.device)
            grown[:, :self.size].copy_(self._archive)
            self._archive = grown
        self._archive[:, self.size].copy_(self.test_bc[:, 0])
        self.size += 1
        self.sizes[self.running] = self.size
        out, thetas = [None] * self.R, None
        for r in np.flatnonzero(self.running):
            mean, ste = np.mean(returns[r]), np.std(returns[r]) / repetitions
            improved = bool(mean > self.best[r])
            if improved:
                thetas = e.theta_numpy() if thetas is None else thetas
                self.best[r], self.best_theta[r] = mean, thetas[r].copy()
            out[r] = (mean, ste, improved)
        return out

    def adapt(self, r, improved):
        """NSRA-ES's schedule of run r's w after its test; a fixed weight stays as it is."""
        if self.adaptive[r]:
            self.reward_weight[r], self.stall[r] = _adapted(self.reward_weight[r], self.stall[r], improved)

    def evaluate(self):
        """Every run's generation: fitness (engine.fitness_all [R, N]) and the members' behaviours (self.bc) from one
        launch (host-stepped: one policy launch per step)."""
        return self.engine.evaluate(bc_out=self.bc)

    def stop(self, r):
        """Run r trains no more: its theta, Adam moments and statistics are kept as they are now."""
        e = self.engine
        self._frozen[r] = {n: None if getattr(e, n) is None else getattr(e, n)[r].clone()
                           for n in ('theta', 'adam_m', 'adam_v', 'obs_stats')}
        self.running[r] = False
        if self.host:
            e.running[r] = False

    def step(self):
        """Every run's novelty against its archive, the blend with its weight w_r (the weight table rewritten when a w
        changed), and the gradient and Adam step of every run."""
        e = self.engine
        self.kn.novelty_runs(self.bc, self._archive, self.k, size=self.size, out=self.novelty)
        if self.reward_weight != self._table_weights:
            self.weight_table.copy_(self.kn.ns_weight_table(self.reward_weight, self.device))
            self._table_weights = list(self.reward_weight)
        self.kn.ns_shape_runs(e.fitness_all, self.novelty, self.weight_table, workspace=self.shape_ws, out=self.shaped)
        for r in np.flatnonzero(self.running):
            self.weights[r].append(self.reward_weight[r])
        e.rank_and_reduce(shaped=self.shaped)
        e.apply()
        e.generation_index += 1


def build_sweep(configs, *, kernels=None, device=None):
    """The NoveltySweep of train_sweep(configs)."""
    return NoveltySweep(configs, kernels=kernels, device=device)


def train_sweep(configs, sweep=None):
    """train(configs[r]) for every r, trained together on one GPU as one sweep: one [training_rewards, training_steps,
    training_timestamps] triple per config, whose rewards and steps are those of train(configs[r]), bit for bit (and so
    are run r's final theta, Adam moments, statistics, archive, weights, best and best_theta: NoveltySweep).  The runs
    share one clock.  The configs may differ in seed, sigma, learning_rate, weight_decay, action_noise_std,
    initial_weight and ns_reward_weight ('adaptive' included), host-stepped ones also in env_fn and batch_env_fn
    (check_sweep_configs).  Closed-loop runs take the same steps and stop together; host-stepped runs count their own
    steps and each stops where its train() would, its environments never reset or stepped again."""
    check_sweep_configs(configs)
    ns = sweep if sweep is not None else build_sweep(configs)
    c, R = configs[0], len(configs)
    reps = c.test_repetitions
    out = [[[], [], []] for _ in range(R)]
    total_steps = np.zeros(R, dtype=np.int64)
    initial_time = time.time()
    iteration = 0
    while True:
        live = np.flatnonzero(ns.running)
        tests = ns.test(reps)
        if iteration > 0:
            for r in live:
                ns.adapt(r, tests[r][2])
        elapsed_time = time.time() - initial_time
        for r in live:
            for log, value in zip(out[r], (tests[r][0], int(total_steps[r]), elapsed_time)):
                log.append(value)
        logger.info('Test: %d runs running, mean %f, elapsed time %d'
                    % (len(live), float(np.mean([out[r][0][-1] for r in live])), elapsed_time))
        fitness = ns.evaluate()
        total_steps[live] += np.broadcast_to(ns.engine.steps_taken, (R,))[live]
        logger.info('Train: iteration %d, mean fitness over %d runs %f'
                    % (iteration, len(live), float(fitness[torch.as_tensor(live)].mean())))
        iteration += 1
        for r in live:                                                  # where train(configs[r]) breaks
            if (c.max_steps and total_steps[r] > c.max_steps) or \
                    (getattr(c, 'max_generations', 0) and iteration > c.max_generations):
                ns.stop(r)
        if not ns.running.any():
            break
        ns.step()
    return out


def multi_runs(config, runs=10, log_dir='log', data_dir='data', batched=False, *, kernels=None, device=None):
    """`runs` train() runs one after the other, run r with seed config.seed + r, with the log file and the pickle of
    [[rewards, steps, timestamps], ...] of natural_es.multi_runs (data/<tag>-stats-<task>.bin, rewritten after every
    run).  batched=True trains them together through train_sweep and writes the same files once: the rewards and steps
    are those of batched=False, bit for bit; the timestamps come from the sweep's one clock.  `kernels` is a stand-in for
    the device ops (ops, or ops_runs when batched)."""
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
            stats = train_sweep(configs, build_sweep(configs, kernels=kernels, device=device))
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
        for run in range(0 if batched else runs):
            c = configs[run]
            logger.info('Run %d' % run)
            stats.append(train(c, build(c, kernels=kernels, device=device)))
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
    finally:
        logger.removeHandler(fh)
        fh.close()
    return stats
