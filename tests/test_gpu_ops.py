"""Parity of the CUDA kernels (through the C ABI) against the oracle on identical seeded inputs.

Layered protocol (SURVEY §8d): noise -> fitness -> ranks -> gradient/update.  Tolerances are stated
next to each assert; integer work (ranks) is bit-exact.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import nes_oracle as orc

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'


def ops():
    from distributedes_b200 import ops as _ops
    return _ops


def relnorm(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def noise_tol(eps_ref):
    """|d eps| bound: 4e-6*(1+|eps|) from MUFU sin/cos/sqrt (abs err 2^-21.4 on the unit circle, times r)
    plus the lg2.approx absolute error 2^-22 which, for u1 -> 1 (r -> 0), turns into 2^-22*ln2/r."""
    return 4e-6 * (1 + np.abs(eps_ref))


@pytest.mark.parametrize('n,P,off,gen', [(3, 4481, 0, 0), (5, 6020, 1000, 7), (2, 73220, 65534, 123456), (4, 10, 0, 1),
                                         (1, 1, 0, 0), (3, 7, 2, 2)])
def test_noise_fill_matches_oracle(n, P, off, gen):
    seed = 0x1234567887654321
    got = ops().noise_fill(n, P, seed, gen, member_offset=off, device=DEV).cpu().numpy().astype(np.float64)
    ref = orc.noise(seed, gen, off, n, P)
    # the small-r clause: r = sqrt(z0^2+z1^2) per Box-Muller pair
    pad = (-P) % 2
    r = np.sqrt((np.pad(ref, ((0, 0), (0, pad))) ** 2).reshape(n, -1, 2).sum(-1)).repeat(2, axis=1)[:, :P]
    tol = noise_tol(ref) + 2.0 ** -22 * np.log(2) / np.maximum(r, 1e-4)
    assert np.all(np.abs(got - ref) <= tol), np.max(np.abs(got - ref) / tol)


def test_noise_statistics_and_empty():
    eps = ops().noise_fill(64, 73220, 99, 3, device=DEV)
    assert abs(eps.mean().item()) < 2e-3 and abs(eps.std().item() - 1) < 2e-3
    assert ops().noise_fill(0, 100, 1, 1, device=DEV).shape == (0, 100)
    assert ops().noise_fill(4, 0, 1, 1, device=DEV).shape == (4, 0)


def test_perturb_matches_oracle():
    d0, H, A = 24, 64, 4
    P = orc.param_count(d0, H, A)
    theta = orc.synthetic_theta(d0, H, A)
    got = ops().nes_perturb(torch.from_numpy(theta).to(DEV), 6, 0.1, 42, 5, member_offset=10).cpu().numpy()
    eps = orc.noise(42, 5, 10, 6, P)
    ref = orc.perturb(theta[None], 0.1, eps)
    r = np.sqrt((eps ** 2).reshape(6, -1, 2).sum(-1)).repeat(2, axis=1)
    tol = 0.1 * (noise_tol(eps) + 2.0 ** -22 * np.log(2) / np.maximum(r, 1e-4)) + 1e-7     # sigma * noise bound + 1 ulp
    assert np.all(np.abs(got.astype(np.float64) - ref) <= tol)


CASES = [  # d0, H, A, T, clip, n_local, offset
    (3, 64, 1, 32, 2.0, 16, 0),        # Pendulum shape, BASELINE configs[0]
    (24, 64, 4, 256, 1.0, 48, 4000),   # configs[1] shape
    (24, 256, 4, 128, 1.0, 12, 65000), # configs[3] shape
    (5, 20, 3, 70, 1.0, 9, 0),         # ragged: nothing a multiple of 4 / 32 / 64
    (24, 64, 4, 1, 1.0, 3, 0),         # single observation
]


@pytest.mark.parametrize('d0,H,A,T,clip,n,off', CASES)
def test_eval_fp32_matches_oracle(d0, H, A, T, clip, n, off):
    obs, target = orc.synthetic_tape(T, d0, A)
    theta = orc.synthetic_theta(d0, H, A)
    seed, gen, sigma = 77, 3, 0.1
    got = ops().nes_eval(torch.from_numpy(theta).to(DEV), torch.from_numpy(obs).to(DEV),
                         torch.from_numpy(target).to(DEV), hidden=H, sigma=sigma, clip=clip, seed=seed,
                         generation=gen, member_offset=off, n_local=n, precision='fp32').cpu().numpy()
    ref = orc.evaluate_population(theta, obs, target, sigma, clip, seed, gen, off, n, d0, H, A)
    # fp32 forward + fp32 noise vs fp64 oracle: relative 2e-5 of |fitness| (measured ~2e-6)
    assert np.max(np.abs(got - ref) / np.abs(ref)) < 2e-5


TC_CASES = [  # d0, H, A, T, clip, n_local, offset
    (24, 64, 4, 256, 1.0, 40, 4000),     # two 128-row tiles on a 2-CTA cluster
    (24, 64, 4, 128, 1.0, 7, 0),
    (24, 128, 4, 256, 1.0, 9, 123),
    (24, 256, 4, 256, 1.0, 10, 65000),   # BASELINE configs[3] shape: one pass on a 2-CTA cluster
    (24, 256, 4, 512, 1.0, 3, 1),
    (8, 64, 2, 128, 2.0, 5, 0),
    (3, 64, 1, 128, 2.0, 6, 0),          # state_dim not a multiple of 4 (generic W1 path)
    (32, 128, 8, 384, 0.5, 4, 9),
]


@pytest.mark.parametrize('precision,tol', [('f16', 4e-3), ('f16x3', 3e-5)])
@pytest.mark.parametrize('d0,H,A,T,clip,n,off', TC_CASES)
def test_eval_tensor_core_matches_oracle(d0, H, A, T, clip, n, off, precision, tol):
    """wgmma forward.  f16: operands rounded to fp16 (2^-11 relative, like TF32) + MUFU tanh.approx (2^-11):
    fitness within 4e-3 relative.  f16x3: hi/lo split operands (~2^-22) + accurate tanh: within 3e-5."""
    obs, target = orc.synthetic_tape(T, d0, A)
    theta = orc.synthetic_theta(d0, H, A)
    seed, gen, sigma = 1234, 5, 0.1
    got = ops().nes_eval(torch.from_numpy(theta).to(DEV), torch.from_numpy(obs).to(DEV),
                         torch.from_numpy(target).to(DEV), hidden=H, sigma=sigma, clip=clip, seed=seed,
                         generation=gen, member_offset=off, n_local=n, precision=precision).cpu().numpy()
    ref = orc.evaluate_population(theta, obs, target, sigma, clip, seed, gen, off, n, d0, H, A)
    err = np.max(np.abs(got - ref) / np.abs(ref))
    assert err < tol, err


def test_eval_tensor_core_many_members_equals_fp32_path():
    """More members than SMs (persistent loop, W2' chunk buffers reused across members): the f16x3
    kernel must agree with the fp32 FFMA kernel member by member."""
    d0, H, A, T, n = 24, 64, 4, 256, 1000
    obs, target = orc.synthetic_tape(T, d0, A)
    th = torch.from_numpy(orc.synthetic_theta(d0, H, A)).to(DEV)
    o, t = torch.from_numpy(obs).to(DEV), torch.from_numpy(target).to(DEV)
    kw = dict(hidden=H, sigma=0.1, clip=1.0, seed=9, generation=2, member_offset=77, n_local=n)
    a = ops().nes_eval(th, o, t, precision='fp32', **kw)
    b = ops().nes_eval(th, o, t, precision='f16x3', **kw)
    c = ops().nes_eval(th, o, t, precision='f16', **kw)
    assert float(((a - b).abs() / a.abs()).max()) < 3e-5
    assert float(((a - c).abs() / a.abs()).max()) < 4e-3
    # deterministic: bit-identical on a second launch
    assert torch.equal(b, ops().nes_eval(th, o, t, precision='f16x3', **kw))


@pytest.mark.parametrize('H,T,precision', [(256, 512, 'f16x3'), (256, 512, 'f16'), (64, 384, 'f16x3'), (256, 384, 'f16x3')])
def test_eval_multi_pass_tile_cache_is_transparent(H, T, precision):
    """Shapes that need several passes over a member: with the optional workspace the weight tiles of pass 0 are
    cached and copied back; without it they are regenerated.  Both must give bit-identical fitness."""
    d0, A, n = 24, 4, 300
    obs, target = orc.synthetic_tape(T, d0, A)
    th = torch.from_numpy(orc.synthetic_theta(d0, H, A)).to(DEV)
    o, t = torch.from_numpy(obs).to(DEV), torch.from_numpy(target).to(DEV)
    ws = ops().eval_workspace(d0, H, A, T, precision, DEV)
    assert ws is not None and ws.numel() > 0
    kw = dict(hidden=H, sigma=0.1, clip=1.0, seed=4, generation=1, member_offset=5, n_local=n, precision=precision)
    a = ops().nes_eval(th, o, t, **kw)
    b = ops().nes_eval(th, o, t, workspace=ws, **kw)
    assert torch.equal(a, b)
    ref = orc.evaluate_population(th.cpu().numpy(), obs, target, 0.1, 1.0, 4, 1, 5, 8, d0, H, A)
    assert np.max(np.abs(b[:8].cpu().numpy() - ref) / np.abs(ref)) < (3e-5 if precision == 'f16x3' else 4e-3)
    assert ops().eval_workspace(d0, 64, A, 256, 'f16', DEV) is None          # single-pass shape: no scratch needed
    assert ops().eval_workspace(d0, 256, A, 256, 'f16x3', DEV) is None       # one pass on a 2-CTA cluster


def test_eval_state_generation_overrides_argument():
    d0, H, A, T = 24, 64, 4, 64
    obs, target = orc.synthetic_tape(T, d0, A)
    theta = torch.from_numpy(orc.synthetic_theta(d0, H, A)).to(DEV)
    o, t = torch.from_numpy(obs).to(DEV), torch.from_numpy(target).to(DEV)
    st = ops().new_state(DEV, generation=9)
    a = ops().nes_eval(theta, o, t, hidden=H, sigma=0.1, clip=1.0, seed=1, generation=0, state=st, n_local=8)
    b = ops().nes_eval(theta, o, t, hidden=H, sigma=0.1, clip=1.0, seed=1, generation=9, n_local=8)
    assert torch.equal(a, b)
    ops().state_advance(st)
    assert ops().read_state(st) == dict(generation=10, adam_t=1, beta1_t=0.9, beta2_t=0.999)


@pytest.mark.parametrize('N', [2, 3, 16, 257, 4096, 65536])
def test_centered_rank_exact(N):
    rs = np.random.RandomState(N)
    f = rs.randn(N).astype(np.float32)
    shaped, ranks = ops().centered_rank(torch.from_numpy(f).to(DEV), return_ranks=True)
    assert np.array_equal(ranks.cpu().numpy(), orc.ranks_stable(f))           # integers: bit exact
    assert np.max(np.abs(shaped.cpu().numpy().astype(np.float64) - orc.fitness_shift(f))) <= 6e-8


def test_centered_rank_ties_nan_zero_and_shards():
    f = np.asarray([1, 1, 1, 0, -0.0, 0.0, np.nan, np.inf, -np.inf, 5, np.nan, 1], dtype=np.float32)
    shaped, ranks = ops().centered_rank(torch.from_numpy(f).to(DEV), return_ranks=True)
    assert np.array_equal(ranks.cpu().numpy(), orc.ranks_stable(f))
    # a shard ranks its members against the whole population
    rs = np.random.RandomState(5)
    f = rs.randn(1000).astype(np.float32)
    f[::7] = f[3]                                                             # heavy ties
    full = orc.ranks_stable(f)
    ft = torch.from_numpy(f).to(DEV)
    for off, n in [(0, 1000), (0, 1), (999, 1), (123, 456), (500, 0)]:
        _, r = ops().centered_rank(ft, member_offset=off, n_local=n, return_ranks=True)
        assert np.array_equal(r.cpu().numpy(), full[off:off + n])
    with pytest.raises(RuntimeError):
        ops().centered_rank(torch.zeros(1, device=DEV))                       # N=1: utils.py:146 divides by 0


@pytest.mark.parametrize('N,kind', [(2049, 'ties'), (8193, 'ties'), (20000, 'equal'), (40001, 'few'), (65536, 'nan'), (300001, 'randn')])
def test_centered_rank_bucket_path_edge_cases(N, kind):
    """The bucketed rank (N > 2048): heavy ties, one bucket holding everything, a handful of distinct values, NaN / inf,
    sizes that are not a multiple of any tile, the 1024-bucket path, and shards against the whole population."""
    rs = np.random.RandomState(N)
    f = rs.randn(N).astype(np.float32)
    if kind == 'ties':
        f[::3] = f[1]
    elif kind == 'equal':
        f[:] = 2.5
    elif kind == 'few':
        f = rs.randint(0, 5, N).astype(np.float32)
    elif kind == 'nan':
        f[rs.randint(0, N, 100)] = np.nan
        f[rs.randint(0, N, 100)] = np.inf
        f[rs.randint(0, N, 100)] = -np.inf
        f[rs.randint(0, N, 100)] = -0.0
        f[rs.randint(0, N, 100)] = 0.0
    full = orc.ranks_stable(f)
    ft = torch.from_numpy(f).to(DEV)
    shaped, r = ops().centered_rank(ft, return_ranks=True)
    assert np.array_equal(r.cpu().numpy(), full)
    assert np.max(np.abs(shaped.cpu().numpy().astype(np.float64) - orc.fitness_shift(f))) <= 6e-8
    for off, n in [(0, 1), (N - 1, 1), (N // 8, N // 8), (N // 2 + 3, 1000)]:
        _, r = ops().centered_rank(ft, member_offset=off, n_local=n, return_ranks=True)
        assert np.array_equal(r.cpu().numpy(), full[off:off + n])


@pytest.mark.parametrize('n_local,P,off', [(16, 4481, 0), (4096, 6020, 0), (300, 73220, 5000), (33, 10, 0), (1, 5, 3)])
def test_grad_partial_matches_oracle(n_local, P, off):
    rs = np.random.RandomState(1)
    shaped = (rs.permutation(n_local) / max(n_local - 1, 1) - 0.5).astype(np.float32)
    seed, gen = 2024, 11
    got = ops().nes_grad_partial(torch.from_numpy(shaped).to(DEV), P, seed=seed, generation=gen,
                                 member_offset=off).cpu().numpy()
    ref = np.zeros(P)
    for s in range(0, n_local, 256):
        n = min(256, n_local - s)
        ref += shaped[s:s + n].astype(np.float64) @ orc.noise(seed, gen, off + s, n, P)
    # both norms of SURVEY §8d(iii); 1e-5 is the north-star bar (measured ~3e-7)
    assert relnorm(got, ref) <= 1e-5
    assert np.max(np.abs(got - ref)) <= 1e-5 * np.max(np.abs(ref))


def test_grad_partial_from_dumped_noise_is_tight():
    """Given the GPU's own eps (dump op), the reduction itself is exact to fp32 summation error."""
    n_local, P = 512, 6020
    rs = np.random.RandomState(2)
    shaped = (rs.permutation(n_local) / (n_local - 1) - 0.5).astype(np.float32)
    eps = ops().noise_fill(n_local, P, 5, 1, device=DEV).cpu().numpy().astype(np.float64)
    got = ops().nes_grad_partial(torch.from_numpy(shaped).to(DEV), P, seed=5, generation=1).cpu().numpy()
    assert relnorm(got, shaped.astype(np.float64) @ eps) <= 2e-6


def test_apply_matches_oracle_three_generations():
    P, N = 6020, 4096
    rs = np.random.RandomState(3)
    theta0 = rs.randn(P).astype(np.float32) * 0.1
    theta = torch.from_numpy(theta0.copy()).to(DEV)
    m = torch.zeros(P, dtype=torch.float64, device=DEV)
    v = torch.zeros(P, dtype=torch.float64, device=DEV)
    st = ops().new_state(DEV)
    upd = torch.empty(P, dtype=torch.float32, device=DEV)
    g64 = torch.empty(P, dtype=torch.float64, device=DEV)
    opt = orc.Adam()
    th_ref = theta0.copy()
    for gen in range(3):
        partial = (rs.randn(P) * N * 0.01).astype(np.float32)
        ops().nes_apply(theta, m, v, torch.from_numpy(partial).to(DEV), N, st, sigma=0.1, learning_rate=0.1,
                        weight_decay=0.005, update_out=upd, grad_out=g64)
        ops().state_advance(st)
        g_ref = partial.astype(np.float64) / N / 0.1
        th_ref, upd_ref = orc.nes_update(th_ref, g_ref, opt, 0.005, 0.1)
        assert relnorm(g64.cpu().numpy(), g_ref) <= 1e-15
        assert relnorm(upd.cpu().numpy(), upd_ref) <= 1e-7          # fp64 Adam on both sides, one fp32 rounding
        assert np.max(np.abs(theta.cpu().numpy() - th_ref)) <= 1e-7
    # fp64 on both sides; CUDA contracts a*b+c into fma, so compare to a few ulps of the largest term
    assert np.max(np.abs(m.cpu().numpy() - opt.m)) <= 1e-14 * np.max(np.abs(opt.m))
    assert np.max(np.abs(v.cpu().numpy() - opt.v)) <= 1e-14 * np.max(np.abs(opt.v))


def test_cpu_tensors_and_bad_shapes_are_errors():
    with pytest.raises(RuntimeError, match='CPU tensor'):
        ops().centered_rank(torch.zeros(8))
    theta = torch.zeros(10, device=DEV)
    with pytest.raises(RuntimeError, match='theta has'):
        ops().nes_eval(theta, torch.zeros(4, 3, device=DEV), torch.zeros(4, 1, device=DEV), hidden=64, sigma=0.1,
                       clip=1.0, seed=0, n_local=1)
    with pytest.raises(RuntimeError, match='needs hidden in'):
        P = orc.param_count(3, 5, 1)
        ops().nes_eval(torch.zeros(P, device=DEV), torch.zeros(4, 3, device=DEV), torch.zeros(4, 1, device=DEV),
                       hidden=5, sigma=0.1, clip=1.0, seed=0, n_local=1, precision='f16')
