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

from .engine import NESEngine, kernels_and_device
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
def multi_runs(config, runs=10, log_dir='log', data_dir='data'):
    """natural_es.py:113-124: `runs` sequential train() runs, a per-task log file and the pickle of
    [[rewards, steps, timestamps], ...] rewritten after every run — same file names and on-disk format as the reference
    (its plotting scripts read data/<tag>-stats-<task>.bin).  Unlike the reference the directories are created, and the
    optimiser state does not leak from one run to the next (natural_es.py:120-122 reuses config.opt)."""
    os.makedirs(log_dir, exist_ok=True)
    os.makedirs(data_dir, exist_ok=True)
    fh = logging.FileHandler(os.path.join(log_dir, '%s-%s.txt' % (config.tag, config.task)))
    fh.setLevel(logging.DEBUG)
    logger.addHandler(fh)
    stats = []
    try:
        for run in range(runs):
            logger.info('Run %d' % (run))
            stats.append(train(config))
            with open(os.path.join(data_dir, '%s-stats-%s.bin' % (config.tag, config.task)), 'wb') as f:
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
