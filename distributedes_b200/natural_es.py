"""NES master loop with the reference's surface (natural_es.py:10-110): Worker / train() / test().

The reference's train() forks `num_workers` CPU processes that pull member indices from a queue, draw
eps, roll out, and pipe (eps, fitness, steps) back (natural_es.py:21-32, 62-73).  Here a Worker is "the
process that owns one GPU and a contiguous shard of the population"; the loop body is
engine.NESEngine.generation().  Launch one process per GPU (torchrun, or `launch()` below) and call
train(config) in each; with torch.distributed uninitialised it is a single-GPU run.
"""
from __future__ import annotations

import logging
import os
import pickle
import time

import numpy as np
import torch
import torch.distributed as dist

from .engine import HostEnvSweepEngine, NESEngine, RolloutRunsEngine, kernels_and_device
from .fitness import from_config
from .utils import Evaluator, SharedStats, StaticNormalizer, logger


class Worker:
    """natural_es.py:10-32 re-cast: owns the shard [offset, offset+n_local) on one GPU.  run() evaluates the
    shard for the current generation and returns its fitnesses (the reference's result_q payload minus eps,
    which is never shipped)."""

    def __init__(self, id, param, state_normalizer, task_q, result_q, stop, config, engine=None):
        self.id = id
        self.param = param
        self.state_normalizer = state_normalizer
        self.task_q, self.result_q, self.stop = task_q, result_q, stop      # kept for signature parity; unused
        self.config = config
        self.engine = engine if engine is not None else build_engine(config, param)

    def run(self):
        e = self.engine
        e.evaluate()
        return e.fitness_all[e.offset:e.offset + e.n_local]


def build_engine(config, param=None, *, kernels=None, device=None, **kw):
    """The NESEngine of a config: its fitness source (fitness.from_config) and its optimiser settings.  `kw` goes to
    NESEngine (process_group, use_graph)."""
    k, dev = kernels_and_device(kernels, device)
    src = from_config(config, k, dev, sigma=float(config.sigma), mirrored=config.mirrored)
    return NESEngine(state_dim=src.d0, hidden=src.H, action_dim=src.A, pop_size=config.pop_size,
                     theta0=config.initial_weight if param is None else np.asarray(param, dtype=np.float32),
                     sigma=config.sigma, learning_rate=config.learning_rate, weight_decay=config.weight_decay,
                     clip=config.clip, beta1=config.opt.beta1, beta2=config.opt.beta2, epsilon=config.opt.epsilon,
                     mirrored=config.mirrored, source=src, kernels=k, device=dev, **kw)


def train(config, engine=None):
    """natural_es.py:34-99.  Returns [training_rewards, training_steps, training_timestamps]."""
    stats = SharedStats(config.state_dim)
    engine = engine if engine is not None else build_engine(config)
    worker = Worker(engine.rank, None, StaticNormalizer(config.state_dim), None, None, None, config, engine=engine)

    training_rewards, training_steps, training_timestamps = [], [], []
    initial_time = time.time()
    total_steps = 0
    iteration = 0
    while True:
        test_mean, test_ste = test(config, None, stats, engine=engine)           # :54
        elapsed_time = time.time() - initial_time
        training_rewards.append(test_mean)
        training_steps.append(total_steps)
        training_timestamps.append(elapsed_time)
        if engine.rank == 0:
            logger.info('Test: total steps %d, %f(%f), elapsed time %d' % (total_steps, test_mean, test_ste, elapsed_time))

        worker.run()                                                           # :62-73 (evaluate + gather)
        rewards = engine.fitness_all
        total_steps += engine.steps_taken                                      # :75, the episodes' real lengths
        r_mean = float(rewards.mean())
        r_std = float(rewards.std(unbiased=False))
        if engine.rank == 0:
            logger.info('Train: iteration %d, %f(%f)' % (iteration, r_mean, r_std / np.sqrt(config.pop_size)))
        iteration += 1
        if config.max_steps and total_steps > config.max_steps:                # :82-84
            break
        if getattr(config, 'max_generations', 0) and iteration > config.max_generations:
            break
        engine.rank_and_reduce()                                               # :90-92
        engine.apply()                                                         # :93-96
        engine.generation_index += 1
    return [training_rewards, training_steps, training_timestamps]


def check_runs_config(config):
    """Raises ValueError unless train_runs can batch runs of `config`: a closed-loop device environment
    (ClosedLoopPendulumConfig), plain sampling, at most 2048 members, one process."""
    if getattr(config, 'host_env', False):
        raise ValueError('train_runs: host-stepped environments are not batched over runs (the device batches its own '
                         'closed-loop environments only: ClosedLoopPendulumConfig); use train()')
    if not getattr(config, 'closed_loop', False):
        raise ValueError('train_runs: tape configs are not batched over runs (the device batches its own closed-loop '
                         'environments only: ClosedLoopPendulumConfig); use train()')
    if config.mirrored:
        raise ValueError('train_runs: mirrored sampling is not batched over runs; use train()')
    if int(config.pop_size) > RolloutRunsEngine.MAX_RUN_SIZE:
        raise ValueError('train_runs: pop_size %d > %d: runs are batched up to %d members (a larger population fills the '
                         'GPU alone); use train()' % (config.pop_size, RolloutRunsEngine.MAX_RUN_SIZE,
                                                      RolloutRunsEngine.MAX_RUN_SIZE))
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        raise ValueError('train_runs: a batch of runs trains on one GPU; the process group has world size %d'
                         % dist.get_world_size())


def build_runs_engine(config, runs, *, kernels=None, device=None, **kw):
    """The RolloutRunsEngine of `runs` runs of a config that check_runs_config accepts, every run starting from
    config.initial_weight (as the reference's multi_runs does).  `kw` goes to RolloutRunsEngine (use_graph)."""
    check_runs_config(config)
    return RolloutRunsEngine(task=config.task, hidden=config.hidden_size, pop_size=config.pop_size, runs=runs,
                             theta0=config.initial_weight, sigma=config.sigma, learning_rate=config.learning_rate,
                             weight_decay=config.weight_decay, repetitions=config.repetitions, clip=config.clip,
                             action_noise_std=config.action_noise_std, normalize_obs=config.normalize_obs,
                             seed=config.seed, beta1=config.opt.beta1, beta2=config.opt.beta2,
                             epsilon=config.opt.epsilon, kernels=kernels, device=device, **kw)


def train_runs(config, runs, engine=None):
    """`runs` independent train(config) runs trained together on one GPU (engine.RolloutRunsEngine): a list of `runs`
    [training_rewards, training_steps, training_timestamps] triples.  Run 0 is train(config), bit for bit; runs 1.. draw
    further independent streams of config.seed (not the runs of other seeds).  The runs share one clock, so they share
    steps and timestamps.  ClosedLoopPendulumConfig only (see check_runs_config)."""
    check_runs_config(config)
    engine = engine if engine is not None else build_runs_engine(config, runs)
    R = engine.R
    rewards, steps, timestamps = [[] for _ in range(R)], [], []
    initial_time = time.time()
    total_steps = 0
    iteration = 0
    while True:
        returns = engine.test_returns(config.test_repetitions)                 # [R, repetitions], one launch
        elapsed_time = time.time() - initial_time
        for r in range(R):
            rewards[r].append(np.mean(returns[r]))                             # test(), natural_es.py:101-110
        steps.append(total_steps)
        timestamps.append(elapsed_time)
        logger.info('Test: total steps %d, mean over %d runs %f, elapsed time %d'
                    % (total_steps, R, float(np.mean([rw[-1] for rw in rewards])), elapsed_time))
        fitness = engine.evaluate()
        total_steps += engine.steps_taken
        logger.info('Train: iteration %d, mean fitness over %d runs %f' % (iteration, R, float(fitness.mean())))
        iteration += 1
        if config.max_steps and total_steps > config.max_steps:
            break
        if getattr(config, 'max_generations', 0) and iteration > config.max_generations:
            break
        engine.rank_and_reduce()
        engine.apply()
        engine.generation_index += 1
    return [[rewards[r], list(steps), list(timestamps)] for r in range(R)]


# The fields every config of a sweep shares: the runs of one RolloutRunsEngine share its shapes, its stopping rule and
# Adam's beta and epsilon (beta^t is in the one des_state).  Only seed, sigma, learning_rate, weight_decay,
# action_noise_std and initial_weight may differ; fields the trainer does not read (tag, ...) are not compared.
SWEEP_SHARED = ('task', 'hidden_size', 'pop_size', 'repetitions', 'test_repetitions', 'clip', 'normalize_obs',
                'opt.beta1', 'opt.beta2', 'opt.epsilon', 'max_steps', 'max_generations')


def _field(config, name):
    value = config
    for part in name.split('.'):
        value = getattr(value, part, None)
    return value


# The fields every host-stepped config of a sweep shares (HostEnvSweepEngine): each run may also have its own env_fn and
# batch_env_fn, and its task names nothing the trainer reads.
SWEEP_HOST_SHARED = ('hidden_size', 'pop_size', 'state_dim', 'action_dim', 'repetitions', 'test_repetitions', 'clip',
                     'normalize_obs', 'opt.beta1', 'opt.beta2', 'opt.epsilon', 'max_steps', 'max_generations')


def _host_sweep(configs):
    """Whether `configs` is a host-stepped sweep; a list that mixes host-stepped and other configs is refused."""
    host = [bool(getattr(c, 'host_env', False)) for c in configs]
    if any(host) and not all(host):
        raise ValueError('train_sweep: configs[%d] is host-stepped and configs[%d] is not; the runs of a sweep are all '
                         'host-stepped (HostEnvConfig) or all closed-loop (ClosedLoopPendulumConfig)'
                         % (host.index(True), host.index(False)))
    return all(host)


def check_host_sweep_config(config):
    """Raises ValueError unless a host-stepped sweep can hold a run of `config`: plain sampling, at most 2048 members,
    one process."""
    if config.mirrored:
        raise ValueError('train_sweep: mirrored sampling is not batched over runs; use train()')
    if int(config.pop_size) > HostEnvSweepEngine.MAX_RUN_SIZE:
        raise ValueError('train_sweep: pop_size %d > %d: runs are batched up to %d members (a larger population fills '
                         'the GPU alone); use train()' % (config.pop_size, HostEnvSweepEngine.MAX_RUN_SIZE,
                                                          HostEnvSweepEngine.MAX_RUN_SIZE))
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        raise ValueError('train_sweep: a sweep trains on one GPU; the process group has world size %d'
                         % dist.get_world_size())


def check_sweep_configs(configs):
    """Raises ValueError unless train_sweep can train `configs` as one sweep: all closed-loop configs that each pass
    check_runs_config and agree on every field of SWEEP_SHARED, or all host-stepped configs that each pass
    check_host_sweep_config and agree on every field of SWEEP_HOST_SHARED.  The first field that differs is named."""
    if not len(configs):
        raise ValueError('train_sweep: no configs')
    host = _host_sweep(configs)
    for c in configs:
        (check_host_sweep_config if host else check_runs_config)(c)
    for i, c in enumerate(configs[1:], 1):
        for name in SWEEP_HOST_SHARED if host else SWEEP_SHARED:
            a, b = _field(configs[0], name), _field(c, name)
            if a != b:
                raise ValueError('train_sweep: configs differ in %s (%r in configs[0], %r in configs[%d]); the runs of a '
                                 'sweep may differ only in seed, sigma, learning_rate, weight_decay, action_noise_std '
                                 'and initial_weight%s' % (name, a, b, i, ' (and, host-stepped, their own env_fn and '
                                                           'batch_env_fn)' if host else ''))


def build_sweep_engine(configs, *, kernels=None, device=None, **kw):
    """The engine of a sweep: run r is train(configs[r])'s run, with its seed, hyper-parameters and initial_weight (and,
    host-stepped, its own environments).  Closed-loop configs give a RolloutRunsEngine (`kw`: use_graph), host-stepped
    ones a HostEnvSweepEngine."""
    check_sweep_configs(configs)
    c = configs[0]
    per_run = dict(theta0=np.stack([np.asarray(x.initial_weight, dtype=np.float32).reshape(-1) for x in configs]),
                   seeds=[x.seed for x in configs], sigma=[x.sigma for x in configs],
                   learning_rate=[x.learning_rate for x in configs], weight_decay=[x.weight_decay for x in configs],
                   action_noise_std=[x.action_noise_std for x in configs])
    shared = dict(hidden=c.hidden_size, pop_size=c.pop_size, runs=len(configs), repetitions=c.repetitions, clip=c.clip,
                  normalize_obs=c.normalize_obs, beta1=c.opt.beta1, beta2=c.opt.beta2, epsilon=c.opt.epsilon,
                  kernels=kernels, device=device)
    if _host_sweep(configs):
        return HostEnvSweepEngine(env_fn=[x.env_fn for x in configs],
                                  batch_env_fn=[getattr(x, 'batch_env_fn', None) for x in configs],
                                  state_dim=c.state_dim, action_dim=c.action_dim, test_repetitions=c.test_repetitions,
                                  **per_run, **shared, **kw)
    return RolloutRunsEngine(task=c.task, **per_run, **shared, **kw)


def train_sweep(configs, engine=None):
    """train(configs[r]) for every r, trained together on one GPU as one sweep: one [training_rewards, training_steps,
    training_timestamps] triple per config, whose rewards and steps are those of train(configs[r]).  The runs share one
    clock.  The configs may differ only in seed, sigma, learning_rate, weight_decay, action_noise_std and initial_weight
    (check_sweep_configs); host-stepped ones also in their env_fn and batch_env_fn.  Closed-loop configs train through
    engine.RolloutRunsEngine with seeds, all runs for the same generations; host-stepped ones through
    engine.HostEnvSweepEngine, where each run counts its own steps and stops where train() would."""
    check_sweep_configs(configs)
    engine = engine if engine is not None else build_sweep_engine(configs)
    if not _host_sweep(configs):
        return train_runs(configs[0], len(configs), engine=engine)   # its loop reads only the fields the configs share
    c, R = configs[0], len(configs)
    out = [[[], [], []] for _ in range(R)]
    total_steps = np.zeros(R, dtype=np.int64)
    initial_time = time.time()
    iteration = 0
    while True:
        live = np.flatnonzero(engine.running)
        returns = engine.test_returns(c.test_repetitions)                   # natural_es.py:54, every running run
        elapsed_time = time.time() - initial_time
        for r in live:
            for log, value in zip(out[r], (np.mean(returns[r]), int(total_steps[r]), elapsed_time)):
                log.append(value)
        logger.info('Test: %d runs running, mean %f, elapsed time %d'
                    % (len(live), float(np.mean([out[r][0][-1] for r in live])), elapsed_time))
        fitness = engine.evaluate()
        total_steps[live] += engine.steps_taken[live]                       # :75, each run's episodes' real lengths
        logger.info('Train: iteration %d, mean fitness over %d runs %f'
                    % (iteration, len(live), float(fitness[torch.as_tensor(live)].mean())))
        iteration += 1
        for r in live:                                                      # :82-84, where train(configs[r]) breaks
            if (c.max_steps and total_steps[r] > c.max_steps) or \
                    (getattr(c, 'max_generations', 0) and iteration > c.max_generations):
                engine.running[r] = False
        if not engine.running.any():
            break
        engine.rank_and_reduce()
        engine.apply()
        engine.generation_index += 1
    return out


def test(config, solution, stats, engine=None):
    """natural_es.py:101-110: mean and 'ste' of test_repetitions noiseless episodes of `solution`
    (None = the engine's current parameters)."""
    if engine is not None:
        rewards = engine.test_returns(solution, config.test_repetitions)
    else:
        normalizer = StaticNormalizer(config.state_dim)
        normalizer.offline_stats.load_state_dict(stats.state_dict())
        evaluator = Evaluator(config, normalizer)
        evaluator.model.set_weight(solution)
        rewards = [evaluator.single_run()[0] for _ in range(config.test_repetitions)]
    return np.mean(rewards), np.std(rewards) / config.test_repetitions


def record(config, solution, stats, engine=None):
    """test() recorded: fitness.Trajectories [test_repetitions, horizon, ...] of the test episodes whose mean
    test(config, solution, stats, engine) reports (solution None = the engine's theta).  Closed-loop device configs only.
    Without an engine the episodes are keyed as the first test() of train() keys them (generation word 0), with the
    statistics `stats` (a SharedStats, its state_dict, or None for none yet); with one, `stats` is not read, as in
    test().  Advances nothing."""
    if not getattr(config, 'closed_loop', False):
        raise ValueError('natural_es.record: episodes are recorded on the device\'s closed-loop environments only '
                         '(ClosedLoopPendulumConfig); a host-stepped environment\'s own code sees every step, and a tape '
                         'has no episodes')
    if engine is not None:
        return engine.record_test_episodes(config.test_repetitions, solution)
    k, dev = kernels_and_device()
    src = from_config(config, k, dev, sigma=float(config.sigma), mirrored=config.mirrored)
    if stats is not None and src.obs_stats is not None:
        st = stats.state_dict() if hasattr(stats, 'state_dict') else stats
        src.obs_stats.copy_(torch.from_numpy(np.concatenate([np.asarray(st[x], dtype=np.float32).reshape(-1)
                                                             for x in ('m', 'v', 'n')])))
    theta = config.initial_weight if solution is None else solution
    theta = torch.as_tensor(np.ascontiguousarray(theta, dtype=np.float32).reshape(-1)).to(dev)
    return src.record(theta, repetitions=config.test_repetitions, noiseless=True, generation=0).episode(0)


def _launch_entry(rank, world_size, config_fn, port, result_path):
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world_size)
    try:
        out = train(config_fn())
        if rank == 0:
            # a file, not a pipe: a SimpleQueue.put() of a long run's result blocks once the 64 KiB pipe buffer is full
            # while the parent is still joining the children
            with open(result_path, 'wb') as f:
                pickle.dump(out, f)
    finally:
        dist.destroy_process_group()


def _free_port():
    import socket
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def launch(config_fn, world_size, port=None):
    """Spawn one process per GPU and run train(config_fn()) in each (the reference's `for w in workers:
    w.start()`, natural_es.py:44-45).  config_fn must be picklable (module-level function); `port` defaults to a
    free one on 127.0.0.1."""
    import tempfile
    import torch.multiprocessing as mp
    port = int(port) if port else _free_port()
    fd, path = tempfile.mkstemp(suffix='.des_result')
    os.close(fd)
    try:
        mp.spawn(_launch_entry, args=(world_size, config_fn, port, path), nprocs=world_size, join=True)
        with open(path, 'rb') as f:
            return pickle.load(f)
    finally:
        os.unlink(path)


# ---- run bookkeeping (natural_es.py:113-124; SURVEY 8f row 4) ----------------------------------------------------------
def multi_runs(config, runs=10, log_dir='log', data_dir='data', batched=False):
    """natural_es.py:113-124: `runs` sequential train() runs, a per-task log file and the pickle of
    [[rewards, steps, timestamps], ...] rewritten after every run — same file names and on-disk format as the reference
    (its plotting scripts read data/<tag>-stats-<task>.bin).  Unlike the reference the directories are created, and the
    optimiser state does not leak from one run to the next (natural_es.py:120-122 reuses config.opt).
    batched=True trains the runs together through train_runs (ClosedLoopPendulumConfig only) and writes the same files
    once: run 0 is the first sequential run, the others are independent streams of the same seed."""
    os.makedirs(log_dir, exist_ok=True)
    os.makedirs(data_dir, exist_ok=True)
    if batched:
        check_runs_config(config)
    fh = logging.FileHandler(os.path.join(log_dir, '%s-%s.txt' % (config.tag, config.task)))
    fh.setLevel(logging.DEBUG)
    logger.addHandler(fh)
    stats = []
    path = os.path.join(data_dir, '%s-stats-%s.bin' % (config.tag, config.task))
    try:
        if batched:
            logger.info('Runs 0-%d, batched' % (runs - 1))
            stats = train_runs(config, runs)
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
        for run in range(0 if batched else runs):
            logger.info('Run %d' % (run))
            stats.append(train(config))
            with open(path, 'wb') as f:
                pickle.dump(stats, f)
    finally:
        logger.removeHandler(fh)
        fh.close()
    return stats


_CKPT_SCALARS = ('sigma', 'lr', 'wd', 'beta1', 'beta2', 'epsilon', 'clip')


def save_checkpoint(engine, path):
    """Everything a run needs to resume: theta, Adam (m, v, beta^t, t), generation counter, observation statistics,
    seed, and the hyper-parameters the run was started with (checked on load).  Plain arrays in an .npz container:
    loading never unpickles.  (The reference keeps no training checkpoint, SURVEY 5.)"""
    from . import ops
    st = ops.read_state(engine.state)
    blob = dict(theta=engine.theta_numpy(), adam_m=engine.adam_m.cpu().numpy(), adam_v=engine.adam_v.cpu().numpy(),
                generation=np.uint64(st['generation']), adam_t=np.uint64(st['adam_t']),
                beta1_t=np.float64(st['beta1_t']), beta2_t=np.float64(st['beta2_t']),
                seed=np.uint64(engine.seed), pop_size=np.int64(engine.N), dims=np.asarray([engine.d0, engine.H, engine.A]),
                precision=np.str_(engine.precision), normalize_obs=np.bool_(engine.normalize_obs),
                mirrored=np.bool_(engine.mirrored),
                hyper=np.asarray([getattr(engine, k) for k in _CKPT_SCALARS], dtype=np.float64))
    if engine.normalize_obs:
        blob['obs_stats'] = engine.obs_stats.cpu().numpy()
    with open(path, 'wb') as f:
        np.savez(f, **blob)


def load_checkpoint(engine, path):
    """Restore a checkpoint written by save_checkpoint into an engine built with the same MLP dims, population,
    precision, normaliser setting and optimiser hyper-parameters (anything else raises: resuming into a different
    configuration would silently continue with inconsistent state)."""
    from ._lib import State
    with np.load(path, allow_pickle=False) as blob:
        if tuple(int(v) for v in blob['dims']) != (engine.d0, engine.H, engine.A) or int(blob['pop_size']) != engine.N:
            raise ValueError('checkpoint is for dims %r / population %r' % (blob['dims'].tolist(), int(blob['pop_size'])))
        if str(blob['precision']) != engine.precision or bool(blob['normalize_obs']) != engine.normalize_obs:
            raise ValueError('checkpoint was written with precision=%s normalize_obs=%s; the engine has %s / %s' %
                             (blob['precision'], bool(blob['normalize_obs']), engine.precision, engine.normalize_obs))
        # checkpoints written before mirrored sampling existed have no key: they are plain runs
        mirrored = bool(blob['mirrored']) if 'mirrored' in blob.files else False
        if mirrored != engine.mirrored:
            raise ValueError('checkpoint was written with mirrored=%s; the engine has mirrored=%s' % (mirrored, engine.mirrored))
        mine = np.asarray([getattr(engine, k) for k in _CKPT_SCALARS], dtype=np.float64)
        if not np.array_equal(mine, blob['hyper']):
            raise ValueError('checkpoint hyper-parameters %r differ from the engine\'s %r (%s)' %
                             (blob['hyper'].tolist(), mine.tolist(), ', '.join(_CKPT_SCALARS)))
        engine.theta.copy_(torch.from_numpy(blob['theta']))
        engine.adam_m.copy_(torch.from_numpy(blob['adam_m']))
        engine.adam_v.copy_(torch.from_numpy(blob['adam_v']))
        raw = bytes(State(int(blob['generation']), int(blob['adam_t']), float(blob['beta1_t']), float(blob['beta2_t'])))
        engine.state.copy_(torch.frombuffer(bytearray(raw), dtype=torch.uint8))
        engine.seed = int(blob['seed'])
        engine.generation_index = int(blob['generation'])
        if engine.normalize_obs:
            engine.obs_stats.copy_(torch.from_numpy(blob['obs_stats']))
