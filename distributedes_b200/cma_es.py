"""CMA-ES with the reference's surface (cma_es.py:13-111): Worker / train() / test(), and the strategy object the
reference takes from the third-party `cma` package (cma.CMAEvolutionStrategy, cma_es.py:49: ask() :62, tell() :90).

The hot arithmetic — the rank-mu covariance update inside tell() — is des_cma_rank_mu + des_cma_cov_apply
(csrc/des_cma.cu); solutions are evaluated through a fitness source (fitness.py) and rank-shaped by
des_centered_rank.  The small O(n)/O(n^2) bookkeeping around it (mean, evolution paths, step size) and the library
calls a CMA step needs (the [lambda,n]x[n,n] sampling GEMM and the symmetric eigendecomposition) go through torch
(cuBLAS / cuSOLVER): plumbing, not kernels of this repo.  Equations: Hansen's tutorial arXiv:1604.00772 (cited at README.md:16);
pycma itself is not available here, so this follows oracle/cma_oracle.py's restatement ("parity unpinned").
"""
from __future__ import annotations

import sys
import time

import numpy as np
import torch

from . import fitness
from .engine import RankGroup, kernels_and_device
from .utils import StaticNormalizer, logger


def cma_constants(n, lam):
    """Default strategy parameters, tutorial Table 1 (positive weights)."""
    wp = np.log((lam + 1) / 2.0) - np.log(np.arange(1, lam + 1))
    mu = lam // 2
    mu_eff = wp[:mu].sum() ** 2 / (wp[:mu] ** 2).sum()
    cc = (4 + mu_eff / n) / (n + 4 + 2 * mu_eff / n)
    c1 = 2.0 / ((n + 1.3) ** 2 + mu_eff)
    cmu = min(1 - c1, 2.0 * (0.25 + mu_eff + 1 / mu_eff - 2) / ((n + 2) ** 2 + mu_eff))
    cs = (mu_eff + 2) / (n + mu_eff + 5)
    ds = 1 + 2 * max(0.0, np.sqrt((mu_eff - 1) / (n + 1)) - 1) + cs
    w = np.zeros(lam)
    w[:mu] = wp[:mu] / wp[:mu].sum()
    return dict(w=w, mu=mu, mu_eff=mu_eff, cc=cc, c1=c1, cmu=cmu, cs=cs, ds=ds)


class CMAEvolutionStrategy:
    """GPU-resident (mu/mu_w, lambda)-CMA-ES.  C is fp32 (the rank-mu kernel's type); the vectors and the
    eigen-system are fp64.

    With torch.distributed initialised the lambda members are sharded contiguously over the ranks (SURVEY 8e): ask()
    returns the rank's own members (z regenerated from the counter stream, so no solution is ever shipped), tell() takes
    the local solutions and the GLOBAL cost vector, forms the rank's partial sum_i w_i y_i y_i^T with des_cma_rank_mu as
    packed upper-triangular tiles and all-reduces them — the one collective BASELINE.json's north_star names for CMA-ES —
    plus the n-vector sum_i w_i y_i.  Every rank then applies the identical update, so the strategy state is never broadcast.

    `kernels` (default: distributedes_b200.ops) exists so the world_size > 1 host logic can run under gloo on CPU in the
    test-suite with an oracle-backed stand-in; the product never runs without the CUDA library."""

    def __init__(self, x0, sigma0, popsize, seed=0, device=None, process_group=None, kernels=None):
        self.kn, self.device = kernels_and_device(kernels, device)
        self.group = RankGroup(process_group)
        self.world, self.rank = self.group.world, self.group.rank
        self.n, self.lam, self.seed = len(x0), int(popsize), int(seed)
        self.offset, self.n_local = self.group.shard(self.lam)
        k = cma_constants(self.n, self.lam)
        self.k = k
        dev, f64 = self.device, torch.float64
        self.w64 = torch.tensor(k['w'], dtype=f64, device=dev)
        self.w32 = self.w64.to(torch.float32).contiguous()
        self.m = torch.tensor(np.asarray(x0, dtype=np.float64), device=dev)
        self.sigma = float(sigma0)
        self.C = torch.eye(self.n, dtype=torch.float32, device=dev)
        self.dC = torch.empty_like(self.C)
        self.pc = torch.zeros(self.n, dtype=f64, device=dev)
        self.ps = torch.zeros(self.n, dtype=f64, device=dev)
        self.B = torch.eye(self.n, dtype=f64, device=dev)
        self.D = torch.ones(self.n, dtype=f64, device=dev)
        self.gen = 0
        self.chiN = np.sqrt(self.n) * (1 - 1.0 / (4 * self.n) + 1.0 / (21 * self.n * self.n))
        # lazy eigendecomposition (tutorial, reference code B.2): B, D are refreshed every 1/((c1+cmu) n 10) generations,
        # at least every generation — which is what lambda ~ n/4 gives at BASELINE configs[2] and [4]
        self.eigen_gap = max(1, int(1.0 / ((k['c1'] + k['cmu']) * self.n * 10.0)))

    def ask(self, z=None):
        """The rank's solutions x_i = m + sigma*B*D*z_i, i in [offset, offset + n_local) (cma_es.py:62; all lambda of
        them on a single GPU).  z defaults to the counter noise stream (Philox, stream tag 1, counter = (j/4, member,
        generation)): a pure function of the member index, so shards regenerate it instead of receiving it."""
        if z is None:
            z = self.kn.noise_fill(self.n_local, self.n, self.seed, self.gen, member_offset=self.offset, stream_tag=1,
                                   device=self.device)
        self.z = z
        BD = (self.B * self.D).to(torch.float32)                 # columns scaled by D
        y = z.to(torch.float32) @ BD.T                           # [n_local, n] x [n, n]  (library GEMM)
        self.X = (self.m + self.sigma * y.to(torch.float64)).to(torch.float32).contiguous()
        self._y_of_X = y          # tell() reuses it: (X - m)/sigma from the fp32-rounded X loses |m|/sigma * 6e-8
        return self.X

    def gather_cost(self, cost_local):
        """[lambda] costs from the ranks' shards: all-reduce of the zero-padded vector (== all-gather, ragged allowed)."""
        cost_local = torch.as_tensor(cost_local, device=self.device, dtype=torch.float32).reshape(-1)
        return self.group.gather(cost_local, self.offset, self.lam)

    def tell(self, solutions, cost):
        """cma_es.py:90.  solutions: the rank's [n_local, n] (as returned by ask; all lambda on a single GPU),
        cost [lambda] GLOBAL (lower is better; rank-shaped or raw — only the order matters)."""
        k, n = self.k, self.n
        cost = torch.as_tensor(cost, device=self.device, dtype=torch.float64).reshape(-1)
        if cost.numel() != self.lam:
            raise ValueError('tell() needs the cost of all %d members (got %d)' % (self.lam, cost.numel()))
        order = torch.sort(cost, stable=True).indices                        # identical on every rank
        X = torch.as_tensor(solutions, device=self.device)
        if X.shape[0] != self.n_local:
            raise ValueError('tell() needs this rank\'s %d solutions (got %d)' % (self.n_local, X.shape[0]))
        # weight of each local member = w[its position in the global order]
        pos = torch.empty_like(order)
        pos[order] = torch.arange(self.lam, device=self.device)
        w_loc64 = self.w64[pos[self.offset:self.offset + self.n_local]]
        if X is getattr(self, 'X', None) and getattr(self, '_y_of_X', None) is not None:
            Y = self._y_of_X.to(torch.float64)                                # exactly the y that ask() sampled
        else:
            Y = (X.to(torch.float64) - self.m) / self.sigma                   # foreign solutions: y_i from x_i
        yw = w_loc64 @ Y if self.n_local else torch.zeros(n, dtype=torch.float64, device=self.device)
        # ---- the hot part: rank-mu partial of the shard on our kernel (fp32), summed over ranks.  Sharded runs keep the
        # partial as packed upper-triangular tiles: the all-reduce moves half the bytes of the [n, n] matrix and the
        # covariance update mirrors the tiles while applying them.
        packed = self.world > 1
        Y32, w32 = Y.to(torch.float32).contiguous(), w_loc64.to(torch.float32).contiguous()
        if packed:
            if getattr(self, 'dC_tiles', None) is None:
                self.dC_tiles = torch.zeros(self.kn.cma_packed_elems(n), dtype=torch.float32, device=self.device)
            if self.n_local:
                self.kn.cma_rank_mu_packed(Y32, w32, out=self.dC_tiles)
            else:
                self.dC_tiles.zero_()
            self.group.sum_(self.dC_tiles)                                    # the CMA collective of north_star
        else:
            if self.n_local:
                self.kn.cma_rank_mu(Y32, w32, out=self.dC)
            else:
                self.dC.zero_()
        self.group.sum_(yw)
        self.m = self.m + self.sigma * yw
        cs, ds, cc, c1, cmu, mu_eff = k['cs'], k['ds'], k['cc'], k['c1'], k['cmu'], k['mu_eff']
        cinv_yw = self.B @ ((self.B.T @ yw) / self.D)
        self.ps = (1 - cs) * self.ps + np.sqrt(cs * (2 - cs) * mu_eff) * cinv_yw
        norm_ps = float(torch.linalg.norm(self.ps))
        hsig = float(norm_ps / np.sqrt(1 - (1 - cs) ** (2 * (self.gen + 1))) / self.chiN < 1.4 + 2.0 / (n + 1))
        self.pc = (1 - cc) * self.pc + hsig * np.sqrt(cc * (2 - cc) * mu_eff) * yw
        decay = 1 + c1 * (1 - hsig) * cc * (2 - cc) - c1 - cmu * float(k['w'].sum())
        pc32 = self.pc.to(torch.float32).contiguous()
        if packed:
            self.kn.cma_cov_apply_packed(self.C, self.dC_tiles, pc32, decay=decay, c1=c1, cmu=cmu)
        else:
            self.kn.cma_cov_apply(self.C, self.dC, pc32, decay=decay, c1=c1, cmu=cmu)
        self.sigma = self.sigma * float(np.exp((cs / ds) * (norm_ps / self.chiN - 1)))
        self.gen += 1
        if self.gen % self.eigen_gap == 0:
            d2, self.B = torch.linalg.eigh(self.C.to(torch.float64))        # library eigendecomposition (cuSOLVER)
            self.D = torch.sqrt(torch.clamp(d2, min=1e-300))
        return order


class Worker:
    """cma_es.py:13-29 re-cast: evaluates the solutions of this rank's shard on one GPU through the fitness source its
    config describes (fitness.from_config), which keeps what the reference's workers share with the master
    (cma_es.py:35-38): the statistics `obs_stats` and the observation totals `obs_totals` of the last evaluation.

    `kernels` (default: distributedes_b200.ops) and `device` exist so the sharded host logic can run under gloo on CPU
    with an oracle-backed stand-in, as in CMAEvolutionStrategy."""

    def __init__(self, id, state_normalizer, task_q, result_q, stop, config, device=None, kernels=None):
        self.id, self.config = id, config
        self.kn, self.device = kernels_and_device(kernels, device)
        self.source = fitness.from_config(config, self.kn, self.device)
        self.obs_stats, self.obs_totals = self.source.obs_stats, self.source.obs_totals
        self.tests_run = 0            # test() calls so far: the generation word of the next test episodes

    def run(self, solutions, member_offset=0, generation=0):
        """cost (cma_es.py:28: Evaluator.eval returns -mean return) of every solution; row i is global member
        member_offset + i of generation `generation` (its reset states, on an environment)."""
        return -self.source.solutions(solutions, offset=member_offset, generation=generation)

    def steps_over_ranks(self, es):
        """Environment steps of the last run(), summed over ranks (cma_es.py:73 sums the episodes' real lengths)."""
        return self.source.steps(es.lam, es.group)

    def test_returns(self, solution, repetitions):
        """Returns of `repetitions` noiseless episodes of one solution (cma_es.py:102-111) with the current statistics.
        The k-th call (k = 0 first) resets its episodes from the test stream with generation word k."""
        ret = self.source.test_returns(solution, int(repetitions), self.tests_run)
        self.tests_run += 1
        return ret

    def merge_obs_stats(self, es):
        """cma_es.py:92-96: the statistics of this generation's observations, summed over ranks, merged into [m|v|n]."""
        self.source.share_totals(es.group)
        self.source.merge(es.lam)


def train(config, worker=None, es=None):
    """cma_es.py:31-100.  Returns [training_rewards, training_steps, training_timestamps].  `worker` / `es` default to a
    Worker and a CMAEvolutionStrategy on the current GPU; pass them to choose the device or the kernels."""
    if worker is None:
        worker = Worker(0, StaticNormalizer(config.state_dim), None, None, None, config)
    if es is None:
        es = CMAEvolutionStrategy(config.initial_weight, config.sigma, config.pop_size, seed=config.seed,
                                  device=worker.device, kernels=worker.kn)
    total_steps = 0
    initial_time = time.time()
    training_rewards, training_steps, training_timestamps = [], [], []
    test_mean, test_ste = test(config, config.initial_weight, None, worker=worker)           # :56
    logger.info('total steps %d, %f(%f)' % (total_steps, test_mean, test_ste))
    training_rewards.append(test_mean)
    training_steps.append(0)
    training_timestamps.append(0)
    generation = 0
    while True:
        solutions = es.ask()                                                                # :62 (this rank's shard)
        cost = es.gather_cost(worker.run(solutions, es.offset, es.gen))                     # :63-72, all lambda costs
        total_steps += worker.steps_over_ranks(es)                                          # :73
        best = int(torch.argmin(cost))                                                      # :75
        elapsed_time = time.time() - initial_time
        best_solution = _fetch_member(es, solutions, best)
        test_mean, test_ste = test(config, best_solution, None, worker=worker)              # :77
        if es.rank == 0:
            logger.info('total steps %d, test %f(%f), best %f, elapased time %f' %
                        (total_steps, test_mean, test_ste, -float(cost.min()), elapsed_time))
        training_rewards.append(test_mean)
        training_steps.append(total_steps)
        training_timestamps.append(elapsed_time)
        generation += 1
        if config.max_steps and total_steps > config.max_steps:                             # :85-87
            break
        if getattr(config, 'max_generations', 0) and generation >= config.max_generations:
            break
        cost32 = cost.to(torch.float32).contiguous()
        shaped = worker.kn.centered_rank(cost32, 0, es.lam, out=torch.empty_like(cost32))   # :89 fitness_shift(cost)
        es.tell(solutions, shaped)                                                          # :90
        worker.merge_obs_stats(es)                                                          # :92-96
    return [training_rewards, training_steps, training_timestamps]


def _fetch_member(es, solutions_local, index):
    """Solution `index` of the global population on every rank: a gather of one row, which its owner holds."""
    i = index - es.offset
    mine = solutions_local[i:i + 1] if 0 <= i < es.n_local else solutions_local[:0]
    return es.group.gather(mine, 0, 1)[0]


def test(config, solution, stats, worker=None):
    """cma_es.py:102-111 (which divides the std by config.repetitions, not test_repetitions).  Closed loop: the mean of
    `test_repetitions` episodes with the worker's current statistics (`stats`, if given, replaces them first)."""
    worker = worker if worker is not None else Worker(0, StaticNormalizer(config.state_dim), None, None, None, config)
    sol = torch.as_tensor(np.asarray(solution.detach().cpu() if isinstance(solution, torch.Tensor) else solution,
                                     dtype=np.float32)).reshape(1, -1).to(worker.device)
    if stats is not None and worker.obs_stats is not None:
        worker.obs_stats.copy_(torch.as_tensor(np.asarray(stats, dtype=np.float32)))
    rewards = worker.test_returns(sol, config.test_repetitions)
    return np.mean(rewards), np.std(rewards) / config.repetitions
