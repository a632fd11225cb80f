"""Runs a function on the ranks of a process group: gloo on the CPU for the tests of the sharded host logic, NCCL (rank r
on cuda:r) for the multi-GPU tests.  The ranks meet through a file store in a fresh temporary directory, so concurrent
runs of the suite never compete for a TCP port."""
import os
import pickle
import tempfile
import time

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _rank(rank, world, tmp, backend, fn, args):
    kw = {}
    if backend == 'nccl':
        torch.cuda.set_device(rank)
        kw['device_id'] = torch.device('cuda', rank)
    else:
        torch.set_num_threads(1)              # the CPU ranks share the host's cores
    dist.init_process_group(backend, init_method='file://' + os.path.join(tmp, 'store'), rank=rank, world_size=world,
                            **kw)
    try:
        res = fn(*args)
        with open(os.path.join(tmp, 'rank%d.pkl' % rank), 'wb') as f:
            pickle.dump(res, f)
    finally:
        dist.destroy_process_group()


def spawn(world, fn, *args, backend='gloo', timeout=600):
    """fn(*args) on each of `world` ranks; returns their return values in rank order.  The ranks are spawned processes
    that start with this process's sys.path, so `fn` must be a module-level function of an importable module (a test
    module is) and `args` must pickle.  Ranks still running after `timeout` seconds are killed, and spawn raises
    TimeoutError: a hung rank fails its test instead of hanging the suite."""
    with tempfile.TemporaryDirectory() as tmp:
        ctx = mp.spawn(_rank, args=(world, tmp, backend, fn, args), nprocs=world, join=False)
        deadline = time.monotonic() + timeout
        try:
            while not ctx.join(timeout=max(deadline - time.monotonic(), 0)):
                if time.monotonic() >= deadline:
                    raise TimeoutError('%s on %d ranks did not finish within %g s' % (fn.__name__, world, timeout))
        finally:
            for p in ctx.processes:
                if p.is_alive():
                    p.kill()
                p.join()
        res = []
        for r in range(world):
            with open(os.path.join(tmp, 'rank%d.pkl' % r), 'rb') as f:
                res.append(pickle.load(f))
        return res
