"""world_size=2 on CPU with gloo: cma_es.CMAEvolutionStrategy sharded over the ranks (members split, z regenerated per
shard, all-reduce of the packed rank-mu partials — the sharded path the GPUs run — and of sum_i w_i y_i) must reproduce the single-process fp64 restatement
(oracle/cma_oracle.CMAState) given the same counter noise."""
import numpy as np
import torch

import cpu_ops
from ranks import spawn

N, LAM, GENS, SEED = 12, 9, 3, 4          # ragged: 5 + 4 members


def _worker():
    from distributedes_b200.cma_es import CMAEvolutionStrategy
    from oracle import cma_oracle as cma
    m0 = np.random.RandomState(0).randn(N)
    es = CMAEvolutionStrategy(m0, 1.0, LAM, seed=SEED, device='cpu', kernels=cpu_ops)
    Xs = []
    for _ in range(GENS):
        X = es.ask()
        Xs.append(X.numpy().copy())
        cost = es.gather_cost(torch.from_numpy(cma.sphere(X.numpy()).astype(np.float32)))
        es.tell(X, cost)
    return dict(m=es.m.numpy(), C=es.C.numpy(), sigma=es.sigma, offset=es.offset, n_local=es.n_local, pc=es.pc.numpy(),
                X=np.stack(Xs))


def test_sharded_cma_with_packed_partials_equals_single_process_restatement():
    from oracle import cma_oracle as cma
    from oracle import nes_oracle as orc
    r = spawn(2, _worker)
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
