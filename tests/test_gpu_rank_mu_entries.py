"""des_cma_rank_mu entry by entry against fp64, at the column scales CMA-ES reaches, on both kernels and both layouts.

The reference is plain: (Y64 w)^T Y64 and S = (|Y64| |w|)^T |Y64| as fp64 matmuls (cuBLAS DGEMM) of the same fp32 Y and
w the kernel reads.  Every entry must lie within oracle/rank_mu_error.py's per-entry bound, which is written in S and
the per-column scales, so a column a thousand times smaller than the others is held to its own relative precision
rather than to the largest entry of dC (tests/test_rank_mu_error_model.py checks the bound itself on the CPU).
Beside that: exact power-of-two equivariance, NaN and inf confined to their row and column, the covariance blend per
entry, and the strategy's tell() with foreign solutions.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import cma_oracle as cma
from oracle import rank_mu_error as rm

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F64 = torch.float64


def gram(A, B):
    """A^T B in fp64 on the device."""
    a = torch.from_numpy(np.ascontiguousarray(A, dtype=np.float64)).to(DEV)
    b = torch.from_numpy(np.ascontiguousarray(B, dtype=np.float64)).to(DEV)
    return (a.T @ b).cpu().numpy()


def weights(lam, kind, n):
    """The strategy's default weights (zero for k >= mu) or active-style negative tails; lambda = 1 keeps one member."""
    if lam == 1:
        return np.array([1.0 if kind == 'default' else -0.3], np.float32)
    return cma.cma_constants(n, lam, active=(kind == 'active'))['w'].astype(np.float32)


def population(lam, n, regime, seed):
    """fp32 Y [lambda, n] with the columns of `regime`."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    Y = torch.randn(lam, n, generator=g, device=DEV, dtype=F64)
    log_uniform = lambda lo, hi: 10.0 ** (lo + (hi - lo) * torch.rand(n, generator=g, device=DEV, dtype=F64))
    if regime == 'x2^-12':
        Y *= 2.0 ** -12
    elif regime == 'x2^18':
        Y *= 2.0 ** 18
    elif regime == 'log_uniform':
        Y *= log_uniform(-4, 4)
    elif regime == 'rotated':
        Q = torch.linalg.qr(torch.randn(n, n, generator=g, device=DEV, dtype=F64))[0]
        Y = (Y * log_uniform(-3, 1)) @ Q.T
    elif regime == 'zero_column':
        Y[:, n // 3] = 0.0
    else:
        assert regime == 'unit', regime
    return Y.to(torch.float32).contiguous()


def unpack(tiles, n):
    """The symmetric [n, n] matrix held by packed upper tiles (tile side 64 up to n = 2048, 128 above): the upper
    entries as stored, mirrored bit for bit."""
    tile = 64 if n <= 2048 else 128
    t = (n + tile - 1) // tile
    v = tiles.view(-1, tile, tile)
    full = torch.zeros(t * tile, t * tile, dtype=tiles.dtype, device=tiles.device)
    idx = 0
    for bi in range(t):
        for bj in range(bi, t):
            full[bi * tile:(bi + 1) * tile, bj * tile:(bj + 1) * tile] = v[idx]
            idx += 1
    assert idx * tile * tile == tiles.numel()
    full = full[:n, :n]
    i = torch.arange(n, device=tiles.device)
    return torch.where(i[:, None] <= i[None, :], full, full.T)


def both_layouts(Y, w):
    from distributedes_b200 import ops
    return ops.cma_rank_mu(Y, w), unpack(ops.cma_rank_mu_packed(Y, w), Y.shape[1])


REGIMES = ('unit', 'x2^-12', 'x2^18', 'log_uniform', 'rotated', 'zero_column')
SHAPES = [(2047, 37), (1000, 1),                                                    # fp32 FFMA (n < 2048)
          (2048, 1), (2048, 64), (2049, 65), (2175, 129), (2176, 1024), (4096, 4096)]   # tensor cores
# (2175, 129): three K stages, so the SYRK's two accumulators sum unequal halves; lambda = 4096 keeps the default
# weights only, whose tail (k just below mu) is ~1e-7.
CASES = [(n, lam, kind) for n, lam in SHAPES for kind in (('default',) if lam == 4096 else ('default', 'active'))]


@pytest.mark.parametrize('regime', REGIMES)
@pytest.mark.parametrize('n,lam,kind', CASES)
def test_rank_mu_every_entry_within_bound(n, lam, kind, regime):
    w32 = weights(lam, kind, n)
    Y = population(lam, n, regime, seed=n * 31 + lam * 7 + len(regime) + len(kind))
    w = torch.from_numpy(w32).to(DEV)
    full, packed = both_layouts(Y, w)
    assert torch.equal(full, full.T)                                  # exactly symmetric
    assert torch.equal(packed, full)                                  # the layouts carry the same numbers
    Yn = Y.cpu().numpy()
    ref, S = rm.reference(Yn, w32, gram)
    B = rm.rank_mu_error_bound(Yn, w32, rm.kernel_for(n), gram, S=S)
    r = rm.worst_ratio(full.cpu().numpy(), ref, B)
    # measured on an H100 (700 W): FFMA 0.16..0.20 at lambda = 37 and up to 0.95 at lambda = 1 (one product, where the
    # bound is just its two fp32 roundings); tensor cores 0.12..0.33 over every shape and regime.  The tensor-core kernel
    # without column scales reached 25 (unit columns, lambda = 1), 290 (one zero column), 1.5e5 (x2^-12), 2.6e5
    # (log-uniform) and inf (x2^18).
    assert r <= 1.0, 'largest |dC - ref| / bound %.3g' % r


@pytest.mark.parametrize('kind', ('default', 'active'))
@pytest.mark.parametrize('n,lam', [(2047, 64), (2048, 64), (4096, 256)])
def test_rank_mu_power_of_two_equivariance_is_exact(n, lam, kind):
    """dC(Y diag(2^s)) == diag(2^s) dC(Y) diag(2^s) bit for bit, s_j in [-20, 20], |y| >= 2^-10 so that no fp32
    product underflows: a power of two must change no rounding in either kernel."""
    g = torch.Generator(device=DEV).manual_seed(n + lam)
    Y = torch.randn(lam, n, generator=g, device=DEV)
    Y = torch.sign(Y) * Y.abs().clamp(min=2.0 ** -10)
    s = torch.randint(-20, 21, (n,), generator=g, device=DEV, dtype=torch.int32)
    pow2 = lambda e: ((e + 127) << 23).view(torch.float32)            # 2^e exactly, from the exponent bits
    w = torch.from_numpy(weights(lam, kind, n)).to(DEV)
    Ys = Y * pow2(s)[None, :]
    outer = pow2(s[:, None] + s[None, :])
    for got, base in zip(both_layouts(Ys, w), both_layouts(Y, w)):
        want = base * outer
        assert torch.equal(got, want), '%d of %d entries differ' % (int((got != want).sum()), n * n)


@pytest.mark.parametrize('bad', (float('nan'), float('inf')))
@pytest.mark.parametrize('n,lam', [(2047, 64), (2048, 64), (2049, 65)])
def test_non_finite_input_stays_in_its_row_and_column(n, lam, bad):
    """Y[k, j] = NaN or inf with w_k != 0: row and column j of dC are non-finite, every other entry is bit-identical
    to the run with Y[k, j] = 0 (a non-finite column maximum must not become a finite column scale)."""
    g = torch.Generator(device=DEV).manual_seed(n)
    Y0 = torch.randn(lam, n, generator=g, device=DEV)
    w = torch.from_numpy(weights(lam, 'active', n)).to(DEV)
    k, j = 3, n // 2 + 5
    assert float(w[k]) != 0.0
    Y0[k, j] = 0.0
    Yb = Y0.clone()
    Yb[k, j] = bad
    i = torch.arange(n, device=DEV)
    line = (i[:, None] == j) | (i[None, :] == j)
    for got, base in zip(both_layouts(Yb, w), both_layouts(Y0, w)):
        assert not bool(torch.isfinite(got[line]).any())
        assert torch.equal(got[~line], base[~line])


@pytest.mark.parametrize('consts', ('strategy', 'strong'))
@pytest.mark.parametrize('n,lam', [(2047, 64), (4481, 64), (2176, 1024)])
def test_covariance_blend_every_entry(n, lam, consts):
    """des_cma_cov_apply and _packed against fp64 decay C + c1 pc pc^T + cmu dC of the fp32 C, pc, dC they read,
    within oracle/rank_mu_error.cov_blend_bound (decay, c1, cmu rounded to fp32 by the kernel, then four roundings)."""
    from distributedes_b200 import ops
    if consts == 'strategy':                      # decay = 1 - ~1e-6 at n = 4481, lambda = 64
        k = cma.cma_constants(n, lam)
        c1, cmu = k['c1'], k['cmu']
        decay = 1 - c1 - cmu * float(k['w'].sum())
    else:
        decay, c1, cmu = 0.9, 0.01, 0.05
    g = torch.Generator(device=DEV).manual_seed(n + lam)
    A = torch.randn(n, n, generator=g, device=DEV, dtype=F64) / np.sqrt(n)
    C0 = (A @ A.T + torch.eye(n, device=DEV, dtype=F64)).to(torch.float32)
    C0 = torch.triu(C0) + torch.triu(C0, 1).T                         # exactly symmetric
    pc = torch.randn(n, generator=g, device=DEV)
    Y = population(lam, n, 'log_uniform', seed=n)
    w = torch.from_numpy(weights(lam, 'active', n)).to(DEV)
    dC = ops.cma_rank_mu(Y, w)
    ref, T = rm.cov_blend_reference(C0.cpu().numpy(), dC.cpu().numpy(), pc.cpu().numpy(), decay, c1, cmu)
    B = rm.cov_blend_bound(T)
    C1 = C0.clone()
    ops.cma_cov_apply(C1, dC, pc, decay=decay, c1=c1, cmu=cmu)
    C2 = C0.clone()
    ops.cma_cov_apply_packed(C2, ops.cma_rank_mu_packed(Y, w), pc, decay=decay, c1=c1, cmu=cmu)
    for C in (C1, C2):
        r = rm.worst_ratio(C.cpu().numpy(), ref, B)
        assert r <= 1.0, 'largest |C - ref| / bound %.3g' % r         # measured 0.72..0.81 on an H100 (700 W)


def test_tell_with_foreign_solutions_meets_the_entry_bound():
    """CMAEvolutionStrategy at n = 2304 (tensor cores), lambda = 64, told foreign solutions X = m + sigma Y whose columns
    have axis-aligned scales log-uniform in [1e-3, 10]: es.dC meets the per-entry bound against fp64 of the Y that
    tell() forms, and C stays finite."""
    from distributedes_b200.cma_es import CMAEvolutionStrategy
    n, lam, sigma = 2304, 64, 0.3
    rs = np.random.RandomState(2304)
    m0 = rs.randn(n)
    es = CMAEvolutionStrategy(m0, sigma, lam, seed=5, device=DEV)
    X = torch.from_numpy((m0 + sigma * rs.randn(lam, n) * 10.0 ** rs.uniform(-3, 1, n)).astype(np.float32)).to(DEV)
    cost = rs.permutation(lam).astype(np.float64)
    m = es.m.clone()
    es.tell(X, torch.from_numpy(cost))
    Y32 = ((X.to(F64) - m) / sigma).to(torch.float32).cpu().numpy()          # the y_i tell() forms from x_i
    rank = np.argsort(np.argsort(cost, kind='stable'), kind='stable')
    w32 = es.w64.cpu().numpy()[rank].astype(np.float32)
    ref, S = rm.reference(Y32, w32, gram)
    B = rm.rank_mu_error_bound(Y32, w32, 'tc', gram, S=S)
    r = rm.worst_ratio(es.dC.cpu().numpy(), ref, B)
    assert r <= 1.0, 'largest |dC - ref| / bound %.3g' % r           # measured 0.27 (55 without column scales)
    assert bool(torch.isfinite(es.C).all())
