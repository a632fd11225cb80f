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
host-stepped configs only (a tape has no episodes), plain sampling, one process."""
from __future__ import annotations

import copy
import time

import numpy as np
import torch
import torch.distributed as dist

from . import natural_es
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
        self._archive = torch.zeros((_INITIAL_CAPACITY, self.d), dtype=torch.float32, device=dev)
        self.size = 0
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
        return self._archive[:self.size]

    def _archive_add(self, row):
        if self.size == self._archive.shape[0]:
            grown = torch.zeros((2 * self.size, self.d), dtype=torch.float32, device=self.device)
            grown[:self.size].copy_(self._archive)
            self._archive = grown
        self._archive[self.size].copy_(row.reshape(-1))
        self.size += 1

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
        if not self.adaptive:
            return
        if improved:
            self.reward_weight, self.stall = min(1.0, self.reward_weight + ADAPT_STEP), 0
        else:
            self.stall += 1
            if self.stall >= ADAPT_PATIENCE:
                self.reward_weight, self.stall = max(0.0, self.reward_weight - ADAPT_STEP), 0

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
