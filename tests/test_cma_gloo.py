"""world_size=2 on CPU with gloo: cma_es.CMAEvolutionStrategy sharded over the ranks (members split, z regenerated per
shard, all-reduce of the packed rank-mu partials — the sharded path the GPUs run — and of sum_i w_i y_i) must reproduce the single-process fp64 restatement
(oracle/cma_oracle.CMAState) given the same counter noise."""
import os
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, LAM, GENS, SEED = 12, 9, 3, 4          # ragged: 5 + 4 members


def _worker(rank, world, port, outdir):
    sys.path.insert(0, REPO)
    sys.path.insert(0, os.path.join(REPO, 'tests'))
    import fake_kernels
    from distributedes_b200.cma_es import CMAEvolutionStrategy
    from oracle import cma_oracle as cma
    torch.set_num_threads(1)
    dist.init_process_group('gloo', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world)
    try:
        m0 = np.random.RandomState(0).randn(N)
        es = CMAEvolutionStrategy(m0, 1.0, LAM, seed=SEED, device='cpu', kernels=fake_kernels)
        Xs = []
        for _ in range(GENS):
            X = es.ask()
            Xs.append(X.numpy().copy())
            cost = es.gather_cost(torch.from_numpy(cma.sphere(X.numpy()).astype(np.float32)))
            es.tell(X, cost)
        np.savez(os.path.join(outdir, 'rank%d.npz' % rank), m=es.m.numpy(), C=es.C.numpy(), sigma=es.sigma,
                 offset=es.offset, n_local=es.n_local, pc=es.pc.numpy(), X=np.stack(Xs))
    finally:
        dist.destroy_process_group()


def test_sharded_cma_with_packed_partials_equals_single_process_restatement():
    from oracle import cma_oracle as cma
    from oracle import nes_oracle as orc
    with tempfile.TemporaryDirectory() as outdir:
        mp.spawn(_worker, args=(2, 29691, outdir), nprocs=2, join=True)
        r = [np.load(os.path.join(outdir, 'rank%d.npz' % k)) for k in range(2)]
    assert int(r[0]['offset']) == 0 and int(r[0]['n_local']) + int(r[1]['n_local']) == LAM
    for k in ('m', 'C', 'sigma', 'pc'):                       # identical update on every rank, no broadcast
        assert np.array_equal(r[0][k], r[1][k]), k
    ref = cma.CMAState(np.random.RandomState(0).randn(N), 1.0, LAM)
    for gen in range(GENS):
        # the ranks' shards tile the population; generation 0 (B = I, D = 1) also equals the restatement's own ask().
        # Later generations are fed the ranks' solutions: x = m + sigma*B*D*z depends on eigenvector signs, on which
        # no two eigensolvers agree.
        X = np.concatenate([r[0]['X'][gen], r[1]['X'][gen]]).astype(np.float64)
        if gen == 0:
            z = orc.noise(SEED, 0, 0, LAM, N, stream=orc.STREAM_CMA_Z).astype(np.float32).astype(np.float64)
            assert np.max(np.abs(ref.ask(z) - X)) <= 2e-6 * np.max(np.abs(X))
        ref.tell(X, cma.sphere(X).astype(np.float32))
    # fp32 C and fp32 sampling on the sharded side vs fp64 restatement
    assert np.linalg.norm(r[0]['C'] - ref.C) <= 2e-5 * np.linalg.norm(ref.C)
    assert np.linalg.norm(r[0]['m'] - ref.m) <= 2e-5 * np.linalg.norm(ref.m)
    assert abs(float(r[0]['sigma']) - ref.sigma) <= 2e-5 * ref.sigma
