"""Runs a function on the gloo ranks of a CPU process group, for the tests of the sharded host logic.  The ranks meet
through a file store in a fresh temporary directory, so concurrent runs of the suite never compete for a TCP port."""
import os
import pickle
import tempfile

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _rank(rank, world, tmp, fn, args):
    torch.set_num_threads(1)
    dist.init_process_group('gloo', init_method='file://' + os.path.join(tmp, 'store'), rank=rank, world_size=world)
    try:
        res = fn(*args)
        with open(os.path.join(tmp, 'rank%d.pkl' % rank), 'wb') as f:
            pickle.dump(res, f)
    finally:
        dist.destroy_process_group()


def spawn(world, fn, *args):
    """fn(*args) on each of `world` gloo ranks; returns their return values in rank order.  The ranks are spawned
    processes that start with this process's sys.path, so `fn` must be a module-level function of an importable module
    (a test module is) and `args` must pickle."""
    with tempfile.TemporaryDirectory() as tmp:
        mp.spawn(_rank, args=(world, tmp, fn, args), nprocs=world, join=True)
        res = []
        for r in range(world):
            with open(os.path.join(tmp, 'rank%d.pkl' % r), 'rb') as f:
                res.append(pickle.load(f))
        return res
