"""CMA-ES rank-mu covariance update: CUDA path vs the fp64 restatement (oracle/cma_oracle.py).
The oracle is parity-UNPINNED (pycma is not available; see its header) — the bar is 1e-5 relative."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import cma_oracle as cma

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def both_norms(got, ref, tol=1e-5):
    got = np.asarray(got, dtype=np.float64)
    assert np.linalg.norm(got - ref) <= tol * np.linalg.norm(ref)
    assert np.max(np.abs(got - ref)) <= tol * np.max(np.abs(ref))


@pytest.mark.parametrize('n,lam', [(1024, 256), (257, 37), (64, 5), (130, 200), (3000, 64), (4096, 1024)])
def test_rank_mu_matches_restatement(n, lam):
    from distributedes_b200 import ops
    rs = np.random.RandomState(n + lam)
    k = cma.cma_constants(n, lam)
    m_old = rs.randn(n)
    X = m_old + 0.7 * rs.randn(lam, n)
    Y, _ = cma.sort_and_scale(X, cma.sphere(X), m_old, 0.7)
    ref = cma.rank_mu_delta(Y, k['w'])
    Yt = torch.from_numpy(Y.astype(np.float32)).to(DEV)
    wt = torch.from_numpy(k['w'].astype(np.float32)).to(DEV)
    dC = ops.cma_rank_mu(Yt, wt)
    got = dC.cpu().numpy()
    assert np.array_equal(got, got.T)                      # exactly symmetric
    both_norms(got, ref)
    # full covariance update with a rank-one term
    C0 = np.eye(n) + 0.01 * np.cov(rs.randn(n, 2 * n))
    C0 = 0.5 * (C0 + C0.T)
    pc = rs.randn(n)
    Cref, decay = cma.cov_update(C0, ref, pc, k['c1'], k['cmu'], k['w'].sum())
    Ct = torch.from_numpy(C0.astype(np.float32)).to(DEV)
    ops.cma_cov_apply(Ct, dC, torch.from_numpy(pc.astype(np.float32)).to(DEV), decay=decay, c1=k['c1'], cmu=k['cmu'])
    both_norms(Ct.cpu().numpy(), Cref)


def test_rank_mu_shards_sum_to_whole_and_active_weights():
    """Population sharding: sum of per-shard partials == whole (the all-reduce contract), and signed weights."""
    from distributedes_b200 import ops
    n, lam = 512, 96
    rs = np.random.RandomState(0)
    k = cma.cma_constants(n, lam, active=True)
    Y = rs.randn(lam, n)
    ref = cma.rank_mu_delta(Y, k['w'])
    Yt = torch.from_numpy(Y.astype(np.float32)).to(DEV)
    wt = torch.from_numpy(k['w'].astype(np.float32)).to(DEV)
    parts = [ops.cma_rank_mu(Yt[a:b].contiguous(), wt[a:b].contiguous()) for a, b in [(0, 24), (24, 48), (48, 96)]]
    both_norms(sum(p.cpu().numpy().astype(np.float64) for p in parts), ref)
    empty = ops.cma_rank_mu(Yt[:0].contiguous(), wt[:0].contiguous())
    assert float(empty.abs().max()) == 0.0


def test_rank_mu_eight_shards_of_baseline_config5():
    """BASELINE configs[4]: n=4096, lambda=1024 split over 8 shards of 128 members; the all-reduce contract is
    sum(partials) == whole, checked here on one GPU by summing the eight partials in fp32 like NCCL would."""
    from distributedes_b200 import ops
    n, lam = 4096, 1024
    rs = np.random.RandomState(8)
    k = cma.cma_constants(n, lam)
    Y = rs.randn(lam, n)
    ref = cma.rank_mu_delta(Y, k['w'])
    Yt = torch.from_numpy(Y.astype(np.float32)).to(DEV)
    wt = torch.from_numpy(k['w'].astype(np.float32)).to(DEV)
    total = torch.zeros((n, n), dtype=torch.float32, device=DEV)
    for r in range(8):
        total += ops.cma_rank_mu(Yt[r * 128:(r + 1) * 128].contiguous(), wt[r * 128:(r + 1) * 128].contiguous())
    both_norms(total.cpu().numpy(), ref)


def test_full_cma_generation_matches_restatement():
    """BASELINE configs[2]: sphere, n=1024, lambda=256, sigma0=1 (cma_es.py:147): three generations of
    distributedes_b200.cma_es.CMAEvolutionStrategy against the fp64 restatement.  Both tell() the SAME solutions
    (sampled by the restatement): x = m + sigma*B*D*z depends on the eigenvectors' signs / rotation inside
    near-degenerate eigenspaces, which no two eigensolvers agree on, so ask() is checked against the strategy's
    own B, D instead."""
    from distributedes_b200.cma_es import CMAEvolutionStrategy
    n, lam = 1024, 256
    rs = np.random.RandomState(0)
    m0 = rs.randn(n)
    es = CMAEvolutionStrategy(m0, 1.0, lam, seed=9, device=DEV)
    ref = cma.CMAState(m0, 1.0, lam)
    for gen in range(3):
        X = es.ask()                                                   # z from the counter noise stream (tag 1)
        z = es.z.cpu().numpy().astype(np.float64)
        B, D = es.B.cpu().numpy(), es.D.cpu().numpy()
        own = es.m.cpu().numpy() + es.sigma * ((z * D) @ B.T)          # eq. 38-40 with the strategy's own eigen-system
        assert np.max(np.abs(X.cpu().numpy() - own)) <= 2e-5 * np.max(np.abs(own))      # fp32 sampling GEMM
        if gen == 0:                                                   # B = I, D = 1: also equals the restatement's ask
            assert np.max(np.abs(X.cpu().numpy() - ref.ask(z))) <= 2e-5 * np.max(np.abs(own))
        Xr = ref.ask(rs.randn(lam, n)).astype(np.float32)              # common solutions, exactly representable in fp32
        cost = cma.sphere(Xr)
        es.tell(torch.from_numpy(Xr).to(DEV), torch.from_numpy(cost))
        ref.tell(Xr.astype(np.float64), cost)
        both_norms(es.dC.cpu().numpy(), ref.dC)
        both_norms(es.C.cpu().numpy(), ref.C)
        assert np.linalg.norm(es.m.cpu().numpy() - ref.m) <= 1e-6 * np.linalg.norm(ref.m)
        assert abs(es.sigma - ref.sigma) <= 1e-6 * ref.sigma
        assert np.linalg.norm(es.pc.cpu().numpy() - ref.pc) <= 1e-6 * np.linalg.norm(ref.pc)
        assert np.linalg.norm(es.ps.cpu().numpy() - ref.ps) <= 1e-4 * np.linalg.norm(ref.ps)   # through fp32 C
        # the eigen-system reproduces C
        Crec = (es.B * es.D ** 2) @ es.B.T
        assert float((Crec - es.C.double()).abs().max()) <= 1e-9
    assert es.sigma < 1.0 and cma.sphere(ref.m[None])[0] < cma.sphere(m0[None])[0]     # it is actually optimising


def test_pop_eval_and_cma_train_surface():
    """des_pop_eval == des_nes_eval(sigma=0) for explicit solutions; cma_es.train keeps the reference's return triple."""
    from distributedes_b200 import cma_es, ops
    from distributedes_b200.config import BipedalWalkerConfig
    from oracle import nes_oracle as orc
    cfg = BipedalWalkerConfig(hidden_size=16, tape_len=64)            # cma_es.py:129 uses hidden 16
    cfg.pop_size, cfg.sigma, cfg.max_generations = 64, 1.0, 3
    env = cfg.env_fn()
    sols = np.stack([cfg.initial_weight + 0.05 * np.random.RandomState(i).randn(len(cfg.initial_weight)) for i in range(5)]).astype(np.float32)
    fit = ops.pop_eval(torch.from_numpy(sols).to(DEV), torch.from_numpy(env.obs).to(DEV), torch.from_numpy(env.target).to(DEV),
                       hidden=16, clip=1.0).cpu().numpy()
    ref = orc.tape_fitness(orc.forward(sols, env.obs, 24, 16, 4), env.target, 1.0)
    assert np.max(np.abs(fit - ref) / np.abs(ref)) < 2e-5
    rewards, steps, stamps = cma_es.train(cfg)
    assert len(rewards) == len(steps) == len(stamps) == 4 and steps[0] == 0 and steps[1] == 64 * 64
    assert np.all(np.isfinite(rewards)) and np.all(np.diff(stamps) >= 0)


@pytest.mark.parametrize('n,lam', [(300, 40), (1024, 64), (2500, 24), (4096, 16)])
def test_packed_rank_mu_and_apply_equal_the_full_matrix_path(n, lam):
    """des_cma_rank_mu(packed) + des_cma_cov_apply_packed (the sharded runs' path: the all-reduce payload is the packed
    upper triangle) produce exactly the C of des_cma_rank_mu + des_cma_cov_apply, and C stays exactly symmetric."""
    from distributedes_b200 import ops
    g = torch.Generator(device='cpu').manual_seed(n)
    Y = torch.randn(lam, n, generator=g).to(DEV)
    w = torch.rand(lam, generator=g).to(DEV)
    pc = torch.randn(n, generator=g).to(DEV)
    A = torch.randn(n, n, generator=g)
    S = A @ A.T / n
    C0 = (0.5 * (S + S.T)).to(DEV).contiguous()               # exactly symmetric input
    C1, C2 = C0.clone(), C0.clone()
    dC = ops.cma_rank_mu(Y, w)
    ops.cma_cov_apply(C1, dC, pc, decay=0.9, c1=0.01, cmu=0.05)
    tiles = ops.cma_rank_mu_packed(Y, w)
    assert tiles.numel() == ops.cma_packed_elems(n)
    ops.cma_cov_apply_packed(C2, tiles, pc, decay=0.9, c1=0.01, cmu=0.05)
    assert torch.equal(C1, C2)
    # without the rank-one term (whose fp32 product (c1 pc_i) pc_j is not symmetric in either path) C stays exactly symmetric
    C3 = C0.clone()
    ops.cma_cov_apply_packed(C3, tiles, None, decay=0.9, c1=0.0, cmu=0.05)
    assert torch.equal(C3, C3.T)


@pytest.mark.parametrize('n,lam', [(2048, 8), (2049, 37), (2500, 130), (4096, 128),       # tensor cores (n >= 2048)
                                   (256, 64), (1000, 130), (2047, 9)])                    # fp32 FFMA (n < 2048)
def test_rank_mu_kernel_picked_by_n_matches_restatement(n, lam):
    """Each rank-mu kernel, reached through its own shapes (split-fp16 wgmma SYRK for n >= 2048, fp32 FFMA below), against
    the fp64 restatement: signed weights, ragged sizes; full and packed outputs carry the same numbers."""
    from distributedes_b200 import ops
    rs = np.random.RandomState(n * 7 + lam)
    Y = rs.randn(lam, n) * (1 + rs.rand(n))                       # columns of different scale
    w = rs.rand(lam) / lam
    w[lam // 2:] *= -0.3                                           # active-CMA style negative weights
    ref = cma.rank_mu_delta(Y, w)
    Yt = torch.from_numpy(Y.astype(np.float32)).to(DEV)
    wt = torch.from_numpy(w.astype(np.float32)).to(DEV)
    full = ops.cma_rank_mu(Yt, wt)
    got = full.cpu().numpy()
    assert np.array_equal(got, got.T)
    ref32 = cma.rank_mu_delta(Yt.cpu().numpy().astype(np.float64), wt.cpu().numpy().astype(np.float64))   # same fp32 inputs
    both_norms(got, ref32)
    both_norms(got, ref, tol=2e-5)                                 # + the fp32 rounding of the inputs themselves
    # packed tiles hold exactly the full matrix's upper entries
    tiles = ops.cma_rank_mu_packed(Yt, wt)
    C1 = torch.zeros((n, n), device=DEV)
    C2 = torch.zeros((n, n), device=DEV)
    ops.cma_cov_apply(C1, full, None, decay=0.0, c1=0.0, cmu=1.0)
    ops.cma_cov_apply_packed(C2, tiles, None, decay=0.0, c1=0.0, cmu=1.0)
    assert torch.equal(C1, C2)
