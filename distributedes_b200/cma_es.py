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
import torch.distributed as dist

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
        cost [lambda] GLOBAL (lower is better; rank-shaped or raw — only the order matters).  The three phases around the
        two kernels are the ones CMASweep runs around its run-batched kernels."""
        order, Y32, w32, yw = self._tell_rank_mu_inputs(solutions, cost)
        # ---- the hot part: rank-mu partial of the shard on our kernel (fp32), summed over ranks.  Sharded runs keep the
        # partial as packed upper-triangular tiles: the all-reduce moves half the bytes of the [n, n] matrix and the
        # covariance update mirrors the tiles while applying them.
        packed = self.world > 1
        if packed:
            if getattr(self, 'dC_tiles', None) is None:
                self.dC_tiles = torch.zeros(self.kn.cma_packed_elems(self.n), dtype=torch.float32, device=self.device)
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
        pc32, decay, norm_ps = self._tell_paths(yw)
        c1, cmu = self.k['c1'], self.k['cmu']
        if packed:
            self.kn.cma_cov_apply_packed(self.C, self.dC_tiles, pc32, decay=decay, c1=c1, cmu=cmu)
        else:
            self.kn.cma_cov_apply(self.C, self.dC, pc32, decay=decay, c1=c1, cmu=cmu)
        self._tell_step(norm_ps)
        return order

    def _tell_rank_mu_inputs(self, solutions, cost):
        """tell() before the rank-mu partial: the order of the costs, the weights of the local members, Y and
        yw = sum_i w_i y_i.  Returns (order, Y fp32, w fp32, yw)."""
        n = self.n
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
        return order, Y.to(torch.float32).contiguous(), w_loc64.to(torch.float32).contiguous(), yw

    def _tell_paths(self, yw):
        """tell() between the rank-mu partial and the covariance update: yw summed over ranks, the mean, p_sigma, hsig,
        p_c and the decay of C.  Returns (p_c fp32, decay, |p_sigma|)."""
        k, n = self.k, self.n
        self.group.sum_(yw)
        self.m = self.m + self.sigma * yw
        cs, ds, cc, c1, cmu, mu_eff = k['cs'], k['ds'], k['cc'], k['c1'], k['cmu'], k['mu_eff']
        cinv_yw = self.B @ ((self.B.T @ yw) / self.D)
        self.ps = (1 - cs) * self.ps + np.sqrt(cs * (2 - cs) * mu_eff) * cinv_yw
        norm_ps = float(torch.linalg.norm(self.ps))
        hsig = float(norm_ps / np.sqrt(1 - (1 - cs) ** (2 * (self.gen + 1))) / self.chiN < 1.4 + 2.0 / (n + 1))
        self.pc = (1 - cc) * self.pc + hsig * np.sqrt(cc * (2 - cc) * mu_eff) * yw
        decay = 1 + c1 * (1 - hsig) * cc * (2 - cc) - c1 - cmu * float(k['w'].sum())
        return self.pc.to(torch.float32).contiguous(), decay, norm_ps

    def _tell_step(self, norm_ps):
        """tell() after the covariance update: the step size, the generation and the lazy eigendecomposition."""
        k = self.k
        self.sigma = self.sigma * float(np.exp((k['cs'] / k['ds']) * (norm_ps / self.chiN - 1)))
        self.gen += 1
        if self.gen % self.eigen_gap == 0:
            d2, self.B = torch.linalg.eigh(self.C.to(torch.float64))        # library eigendecomposition (cuSOLVER)
            self.D = torch.sqrt(torch.clamp(d2, min=1e-300))


class CMASweep:
    """R CMA-ES strategies trained as one batch on one GPU (train_sweep): strategy r is the CMAEvolutionStrategy of
    train(configs[r]) (x0, sigma0, lambda, its seed), and its state stays bit-equal to that run's.  The runs share lambda
    and n.  Each strategy's C and dC are views into stacked [R, n, n] tensors, so that one des_cma_rank_mu_runs and one
    des_cma_cov_apply_runs serve every run, and ask()'s normals of every run are one des_noise_fill_sweep (stream 1,
    member_offset 0, under each run's seed: the hp table).  The library calls each run's train() makes stay per run: the
    sampling GEMM of ask, the fp64 vector bookkeeping of tell and the eigendecomposition.

    `running` [R] says which runs still train (train_sweep clears a run's entry where its train() would stop): stopped
    runs are neither asked nor told, and stop(r) detaches their C and dC from the stacked tensors, which the batched
    kernels keep writing, so that a stopped run's reported state is its state at its stop."""

    def __init__(self, x0s, sigma0s, popsize, hp, device=None, kernels=None):
        from . import ops_runs
        self.kn, self.device = kernels_and_device(ops_runs if kernels is None else kernels, device)
        self.hp, self.R, self.lam = hp, len(x0s), int(popsize)
        self.es = [CMAEvolutionStrategy(x0, s0, self.lam, seed=0, device=self.device, kernels=self.kn)
                   for x0, s0 in zip(x0s, sigma0s)]
        es0, R, lam = self.es[0], self.R, self.lam
        self.n, self.k = es0.n, es0.k
        dev, n = self.device, self.n
        self.C = torch.eye(n, dtype=torch.float32, device=dev).repeat(R, 1, 1)
        self.dC = torch.empty_like(self.C)
        for r, es in enumerate(self.es):
            es.C, es.dC = self.C[r], self.dC[r]
        self.X = torch.empty((R, lam, n), dtype=torch.float32, device=dev)
        self.Y = torch.zeros((R, lam, n), dtype=torch.float32, device=dev)
        self.w = torch.zeros((R, lam), dtype=torch.float32, device=dev)
        self.pc = torch.zeros((R, n), dtype=torch.float32, device=dev)
        self.decay = np.ones(R)
        self.running = np.ones(R, dtype=bool)
        self.gen = 0

    def ask(self):
        """[R * lambda, n] fp32: run r's rows r*lambda .. are es[r].ask() (a running run's; a stopped run's rows are
        stale), from one des_noise_fill_sweep."""
        R, lam, n = self.R, self.lam, self.n
        z = self.kn.noise_fill_sweep(self.hp, lam, n, self.gen, stream_tag=1).reshape(R, lam, n)
        for r in np.flatnonzero(self.running):
            # a tensor of its own, as a run's own z is: the sampling GEMM then sees the allocator's alignment whatever
            # lambda * n is, so cuBLAS picks the algorithm train() gets
            self.X[r] = self.es[r].ask(z=z[r].clone())
        return self.X.reshape(R * lam, n)

    def tell(self, shaped, mark=None):
        """tell() of every running run with its row of shaped [R, lambda], around one des_cma_rank_mu_runs and one
        des_cma_cov_apply_runs.  `mark`, if given, is called with the name of each phase as it ends: 'update' after the
        covariance update, 'eigh' after each run's step size and lazy eigendecomposition (scripts/time_cma_sweep.py)."""
        live = np.flatnonzero(self.running)
        state = {}
        for r in live:
            es = self.es[r]
            order, Y32, w32, yw = es._tell_rank_mu_inputs(es.X, shaped[r])
            self.Y[r], self.w[r] = Y32, w32
            state[r] = yw
        self.kn.cma_rank_mu_runs(self.Y, self.w, out=self.dC)
        for r in live:
            pc32, self.decay[r], state[r] = self.es[r]._tell_paths(state[r])
            self.pc[r] = pc32
        decay = torch.as_tensor(self.decay, dtype=torch.float64).to(self.device)
        self.kn.cma_cov_apply_runs(self.C, self.dC, self.pc, decay, c1=self.k['c1'], cmu=self.k['cmu'])
        if mark is not None:
            mark('update')
        for r in live:
            self.es[r]._tell_step(state[r])
        self.gen += 1
        if mark is not None:
            mark('eigh')

    def stop(self, r):
        """Run r trains no more: its C and dC leave the stacked tensors, frozen as they are."""
        self.running[r] = False
        es = self.es[r]
        es.C, es.dC = es.C.clone(), es.dC.clone()


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

    def _recorder(self):
        if not isinstance(self.source, fitness.DeviceRollouts):
            raise TypeError('%s: episodes are recorded on the device\'s closed-loop environments only (DeviceRollouts); '
                            'a host-stepped environment\'s own code sees every step, and a tape has no episodes'
                            % type(self.source).__name__)
        return self.source

    def record_test_episodes(self, solution, repetitions=None):
        """fitness.Trajectories [repetitions, horizon, ...] of the test episodes the next test_returns(solution,
        repetitions) runs (generation word tests_run; repetitions default to the config's test_repetitions, as test()
        runs them): its returns are that call's.  Advances nothing, tests_run included."""
        src = self._recorder()
        sol = torch.as_tensor(np.asarray(solution.detach().cpu() if isinstance(solution, torch.Tensor) else solution,
                                         dtype=np.float32)).reshape(-1).to(self.device)
        reps = repetitions or getattr(self.config, 'test_repetitions', None) or src.test_repetitions
        return src.record(sol, repetitions=int(reps), noiseless=True, generation=self.tests_run).episode(0)

    def record_solutions(self, solutions, member_offset=0, generation=0):
        """fitness.Trajectories [n, repetitions, horizon, ...] of the episodes run(solutions, member_offset, generation)
        runs: -mean of each row's returns, summed in fp64, is its cost bit for bit.  Advances nothing."""
        rows = torch.as_tensor(solutions).to(device=self.device, dtype=torch.float32).contiguous()
        return self._recorder().record(rows, member_offset=member_offset, generation=generation)

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


# ---- sweeps: R CMA-ES runs of different configs trained together on one GPU -------------------------------------------
# The fields every config of a CMA-ES sweep shares (closed-loop, or host-stepped with state_dim / action_dim for task).
# seed, sigma (sigma0), action_noise_std and initial_weight (x0) may differ, and host-stepped configs may have their own
# env_fn and batch_env_fn; learning_rate and weight_decay are not read by CMA-ES.
SWEEP_SHARED = ('task', 'hidden_size', 'pop_size', 'repetitions', 'test_repetitions', 'clip', 'normalize_obs', 'max_steps',
                'max_generations')
SWEEP_HOST_SHARED = ('hidden_size', 'pop_size', 'state_dim', 'action_dim', 'repetitions', 'test_repetitions', 'clip',
                     'normalize_obs', 'max_steps', 'max_generations')
MAX_SWEEP_POP = 2048      # the counting rank of des_centered_rank_runs (larger runs are DES_ERR_UNSUPPORTED)


def check_sweep_configs(configs):
    """Raises ValueError unless train_sweep can train `configs` as one sweep: all closed-loop (ClosedLoopPendulumConfig)
    or all host-stepped (HostEnvConfig) configs of 2 .. 2048 members, in one process, that agree on every field of
    SWEEP_SHARED (closed-loop) or SWEEP_HOST_SHARED (host-stepped).  The first field that differs is named."""
    from .natural_es import _field, _host_sweep
    if not len(configs):
        raise ValueError('cma_es.train_sweep: no configs')
    host = _host_sweep(configs)
    for i, c in enumerate(configs):
        if not host and not getattr(c, 'closed_loop', False):
            raise ValueError('cma_es.train_sweep: configs[%d] is a tape config; tape configs are not batched over runs '
                             '(closed-loop ClosedLoopPendulumConfig or host-stepped HostEnvConfig only); use train()' % i)
        if int(c.pop_size) < 2:
            raise ValueError('cma_es.train_sweep: pop_size %d < 2: the centered rank of des_centered_rank_runs divides by '
                             'pop_size - 1' % c.pop_size)
        if int(c.pop_size) > MAX_SWEEP_POP:
            raise ValueError('cma_es.train_sweep: pop_size %d > %d: the runs of a sweep are ranked by the counting rank of '
                             'des_centered_rank_runs, which takes up to %d members (DES_ERR_UNSUPPORTED); use train()'
                             % (c.pop_size, MAX_SWEEP_POP, MAX_SWEEP_POP))
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        raise ValueError('cma_es.train_sweep: a sweep trains on one GPU; the process group has world size %d'
                         % dist.get_world_size())
    for i, c in enumerate(configs[1:], 1):
        for name in SWEEP_HOST_SHARED if host else SWEEP_SHARED:
            a, b = _field(configs[0], name), _field(c, name)
            if a != b:
                raise ValueError('cma_es.train_sweep: configs differ in %s (%r in configs[0], %r in configs[%d]); the runs '
                                 'of a CMA-ES sweep may differ only in seed, sigma, action_noise_std and initial_weight%s'
                                 % (name, a, b, i, ' (and, host-stepped, their own env_fn and batch_env_fn)' if host
                                    else ''))


class SweepWorker:
    """Worker for every run of a sweep: evaluates each run's solutions through one sweep source (fitness.DeviceSweep
    closed-loop, fitness.HostSweep host-stepped) under its row of the table `hp` (its seed and action noise), and holds
    each run's statistics obs_stats and observation totals obs_totals [R, 2*d0+1].  tests_run counts the test() calls,
    the generation word of the next test episodes, as Worker's does."""

    def __init__(self, configs, device=None, kernels=None):
        from . import ops_runs
        self.kn, self.device = kernels_and_device(ops_runs if kernels is None else kernels, device)
        c, R = configs[0], len(configs)
        self.R, self.host = R, bool(getattr(c, 'host_env', False))
        self.hp = self.kn.run_table([x.seed for x in configs], [x.sigma for x in configs], 0.0, 0.0,
                                    [float(x.action_noise_std) for x in configs], self.device, runs=R)
        shared = dict(hidden=c.hidden_size, repetitions=c.repetitions, clip=c.clip, normalize_obs=c.normalize_obs)
        if self.host:
            self.source = fitness.HostSweep(self.kn, self.device, state_dim=c.state_dim, action_dim=c.action_dim,
                                            test_repetitions=c.test_repetitions,
                                            runs=[dict(env_fn=x.env_fn, batch_env_fn=getattr(x, 'batch_env_fn', None),
                                                       seed=x.seed, sigma=None,
                                                       action_noise_std=float(x.action_noise_std)) for x in configs],
                                            **shared)
        else:
            self.source = fitness.DeviceSweep(self.kn, self.device, runs=R, task=c.task, **shared)
        self.obs_stats, self.obs_totals = self.source.obs_stats, self.source.obs_totals
        self.tests_run = 0
        self.fitness = None
        self.task, self.run_keys = getattr(c, 'task', None), [(x.seed, float(x.action_noise_std)) for x in configs]
        self.test_repetitions = c.test_repetitions

    def run(self, rows, generation, running):
        """cost [R, lambda] (-mean return, cma_es.py:28) of every run's solutions rows [R * lambda, n]."""
        lam = rows.shape[0] // self.R
        if self.fitness is None or self.fitness.shape[1] != lam:
            self.fitness = torch.zeros((self.R, lam), dtype=torch.float32, device=self.device)
        self.source.solutions(rows, self.hp, generation=generation, running=running, out=self.fitness)
        return -self.fitness

    def steps(self, lam):
        """[R] environment steps of the last run() (cma_es.py:73: the episodes' real lengths)."""
        return self.source.steps(lam) if not self.host else np.asarray(self.source.last_steps, dtype=np.int64)

    def test_returns(self, solutions, repetitions, running):
        """[R, repetitions] returns of noiseless episodes of solutions[r] (Worker.test_returns of every running run)."""
        ret = self.source.test_returns(solutions, self.hp, int(repetitions), self.tests_run, running)
        self.tests_run += 1
        return ret

    def record_test_episodes(self, solution, run, repetitions=None):
        """fitness.Trajectories [repetitions, horizon, ...] of run `run`'s test episodes of `solution` as the next
        test_returns runs them: Worker.record_test_episodes under the run's seed and action noise, at member offset 0,
        with its statistics.  Its returns are that call's row `run`.  Advances nothing."""
        if self.host:
            raise TypeError('SweepWorker: episodes are recorded on the device\'s closed-loop environments only; a '
                            'host-stepped environment\'s own code sees every step')
        r = int(run)
        if not 0 <= r < self.R:
            raise ValueError('record_test_episodes: run %r is not in [0, %d)' % (run, self.R))
        s = self.source
        seed, noise = self.run_keys[r]
        src = fitness.DeviceRollouts(self.kn, self.device, task=self.task, hidden=s.H, repetitions=s.repetitions,
                                     clip=s.clip, horizon=s.horizon, action_noise_std=noise, seed=seed,
                                     normalize_obs=s.normalize_obs, sigma=None, mirrored=False)
        src.obs_stats = None if self.obs_stats is None else self.obs_stats[r]      # a view: the run's statistics now
        sol = torch.as_tensor(np.asarray(solution.detach().cpu() if isinstance(solution, torch.Tensor) else solution,
                                         dtype=np.float32)).reshape(-1).to(self.device)
        return src.record(sol, repetitions=int(repetitions or self.test_repetitions), noiseless=True,
                          generation=self.tests_run).episode(0)

    def merge_obs_stats(self, running):
        """Worker.merge_obs_stats of every running run; a stopped run's statistics stay as they were at its stop."""
        if self.obs_stats is None:
            return
        stopped = torch.as_tensor(np.flatnonzero(~np.asarray(running)), device=self.device)
        frozen = self.obs_stats[stopped].clone()
        self.kn.obs_stats_merge_totals_runs(self.obs_stats, self.obs_totals, self.source.d0)
        self.obs_stats[stopped] = frozen


def build_sweep(configs, *, kernels=None, device=None):
    """The (SweepWorker, CMASweep) pair of train_sweep(configs): run r has configs[r]'s seed, sigma0, action noise, x0
    and, host-stepped, its own environments."""
    check_sweep_configs(configs)
    worker = SweepWorker(configs, device=device, kernels=kernels)
    es = CMASweep([x.initial_weight for x in configs], [x.sigma for x in configs], configs[0].pop_size, worker.hp,
                  device=worker.device, kernels=worker.kn)
    return worker, es


def train_sweep(configs, worker=None, es=None):
    """train(configs[r]) for every r, trained together on one GPU: one [training_rewards, training_steps,
    training_timestamps] triple per config, whose rewards and steps are those of train(configs[r]), bit for bit (and so
    is each run's final strategy state es.es[r] and statistics worker.obs_stats[r]).  The runs share one clock.  The
    configs may differ only in seed, sigma, action_noise_std and initial_weight (check_sweep_configs); host-stepped ones
    also in env_fn and batch_env_fn.  Closed-loop runs all take the same steps and stop together; host-stepped runs
    count their own steps and each stops where its train() would, its environments never reset or stepped again."""
    check_sweep_configs(configs)
    if worker is None or es is None:
        worker, es = build_sweep(configs)
    c, R, lam = configs[0], len(configs), es.lam
    out = [[[], [], []] for _ in range(R)]
    total_steps = np.zeros(R, dtype=np.int64)
    initial_time = time.time()
    x0 = torch.from_numpy(np.stack([np.asarray(x.initial_weight, dtype=np.float32).reshape(-1) for x in configs]))
    returns = worker.test_returns(x0.to(worker.device), c.test_repetitions, es.running)           # :56
    for r in range(R):
        for log, value in zip(out[r], (np.mean(returns[r]), 0, 0)):
            log.append(value)
    logger.info('total steps 0, mean over %d runs %f' % (R, float(np.mean([o[0][-1] for o in out]))))
    generation = 0
    while True:
        live = np.flatnonzero(es.running)
        rows = es.ask()                                                                     # :62
        cost = worker.run(rows, es.gen, es.running)                                         # :63-72, [R, lambda]
        total_steps[live] += worker.steps(lam)[live]                                        # :73
        best = torch.argmin(cost, dim=1)                                                    # :75
        elapsed_time = time.time() - initial_time
        best_rows = rows.reshape(R, lam, -1)[torch.arange(R, device=rows.device), best].contiguous()
        returns = worker.test_returns(best_rows, c.test_repetitions, es.running)           # :77
        for r in live:
            for log, value in zip(out[r], (np.mean(returns[r]), int(total_steps[r]), elapsed_time)):
                log.append(value)
        logger.info('%d runs running, total steps %s, mean test %f, elapased time %f'
                    % (len(live), total_steps[live].tolist(), float(np.mean([out[r][0][-1] for r in live])),
                       elapsed_time))
        generation += 1
        for r in live:                                                                      # :85-87, where train() breaks
            if (c.max_steps and total_steps[r] > c.max_steps) or \
                    (getattr(c, 'max_generations', 0) and generation >= c.max_generations):
                es.stop(r)
        if not es.running.any():
            break
        shaped = worker.kn.centered_rank_runs(cost.to(torch.float32).contiguous())          # :89 fitness_shift(cost)
        es.tell(shaped)                                                                     # :90
        worker.merge_obs_stats(es.running)                                                  # :92-96
    return out


def multi_runs(config, runs=10, log_dir='log', data_dir='data', batched=False):
    """The reference's CMA-ES driver (cma_es.py:113-152, natural_es.py:113-124's bookkeeping): `runs` train() runs, a
    per-task log file and the pickle of [[rewards, steps, timestamps], ...] rewritten after every run, with the file names
    and on-disk format of natural_es.multi_runs (data/<tag>-stats-<task>.bin).  Run r uses seed config.seed + r, so the
    runs are independent, as the reference's OS-seeded ones are.  batched=True trains them together through train_sweep
    and writes the same files once: the rewards and steps are those of batched=False, bit for bit; the timestamps come
    from the sweep's one clock.  Unlike natural_es.multi_runs(batched=True), whose runs 1.. are further streams of one
    seed that no single train() reproduces, every run here is a sweep run of its own seed, and so reproducible alone."""
    import copy
    import logging
    import os
    import pickle
    os.makedirs(log_dir, exist_ok=True)
    os.makedirs(data_dir, exist_ok=True)
    configs = []
    for r in range(runs):
        c = copy.copy(config)
        c.seed = config.seed + r
        configs.append(c)
    if batched:
        check_sweep_configs(configs)
    fh = logging.FileHandler(os.path.join(log_dir, '%s-%s.txt' % (config.tag, config.task)))
    fh.setLevel(logging.DEBUG)
    logger.addHandler(fh)
    stats = []
    path = os.path.join(data_dir, '%s-stats-%s.bin' % (config.tag, config.task))
    try:
        if batched:
            logger.info('Runs 0-%d, batched' % (runs - 1))
            stats = train_sweep(configs)
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
        for run in range(0 if batched else runs):
            logger.info('Run %d' % (run))
            stats.append(train(configs[run]))
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
    finally:
        logger.removeHandler(fh)
        fh.close()
    return stats


def _fetch_member(es, solutions_local, index):
    """Solution `index` of the global population on every rank: a gather of one row, which its owner holds."""
    i = index - es.offset
    mine = solutions_local[i:i + 1] if 0 <= i < es.n_local else solutions_local[:0]
    return es.group.gather(mine, 0, 1)[0]


def record(config, solution, stats, worker=None):
    """test() recorded: fitness.Trajectories [test_repetitions, horizon, ...] of the test episodes whose mean test(config,
    solution, stats, worker) reports, with the same statistics (`stats`, if given, replaces the worker's first, as in
    test()).  Closed-loop device configs only.  Without a worker the episodes are keyed as the first test() of train()
    keys them.  Advances nothing."""
    if not getattr(config, 'closed_loop', False):
        raise ValueError('cma_es.record: episodes are recorded on the device\'s closed-loop environments only '
                         '(ClosedLoopPendulumConfig); a host-stepped environment\'s own code sees every step, and a tape '
                         'has no episodes')
    worker = worker if worker is not None else Worker(0, StaticNormalizer(config.state_dim), None, None, None, config)
    if stats is not None and worker.obs_stats is not None:
        worker.obs_stats.copy_(torch.as_tensor(np.asarray(stats, dtype=np.float32)))
    return worker.record_test_episodes(solution, config.test_repetitions)


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
