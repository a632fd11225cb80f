"""The error model behind tests/test_gpu_rank_mu_entries.py, checked on the CPU.

oracle/rank_mu_error.py bounds |dC_kernel - dC_exact| entry by entry for both rank-mu kernels.  Here: the bound holds
for an emulation of each kernel's operand rounding over the column regimes the GPU tests use, it is not vacuous, it is
scale-covariant, and it rejects the tensor-core split without column scales and a single wrong entry — which is what
gives the GPU tests their teeth.
"""
import numpy as np
import pytest

from oracle import cma_oracle as cma
from oracle import rank_mu_error as rm

REGIMES = ('unit', 'x2^-12', 'x2^18', 'log_uniform', 'rotated', 'zero_column')


def weights(lam, kind, n=160):
    """The strategy's default weights (zero for k >= mu) or active-style negative tails; lambda = 1 keeps one member."""
    if lam == 1:
        return np.array([1.0 if kind == 'default' else -0.3], np.float32)
    return cma.cma_constants(n, lam, active=(kind == 'active'))['w'].astype(np.float32)


def population(rs, lam, n, regime):
    Y = rs.randn(lam, n)
    if regime == 'x2^-12':
        Y *= 2.0 ** -12
    elif regime == 'x2^18':
        Y *= 2.0 ** 18
    elif regime == 'log_uniform':
        Y *= 10.0 ** rs.uniform(-4, 4, n)
    elif regime == 'rotated':
        Q = np.linalg.qr(rs.randn(n, n))[0]
        Y = (Y * 10.0 ** rs.uniform(-3, 1, n)) @ Q.T
    elif regime == 'zero_column':
        Y[:, n // 3] = 0.0
    return Y.astype(np.float32)


CASES = [(160, lam, kind) for lam in (1, 37, 129) for kind in ('default', 'active')] + [(48, 4096, 'default')]

# max(bound) / max(emulated error) over REGIMES: ffma 1.6..4.6 (lambda = 1), 12..41 (37), 22..98 (129), 71..674 (4096);
# tc 12..40, 23..79, 47..457, 1.7e3..3.2e3.  The bound adds worst cases over lambda terms where the real errors partly
# cancel, and its wgmma term (384 instructions per K half at lambda = 4096) covers an accumulation the emulation does
# not have, so the factor grows with lambda; the caps catch a bound that has stopped tracking the error at all.
VACUITY_CAP = {'ffma': 2e3, 'tc': 1e4}


@pytest.mark.parametrize('regime', REGIMES)
@pytest.mark.parametrize('n,lam,kind', CASES)
@pytest.mark.parametrize('kernel', ('ffma', 'tc'))
def test_emulated_error_within_bound_and_bound_not_vacuous(kernel, n, lam, kind, regime):
    rs = np.random.RandomState(lam * 7 + len(regime))
    Y, w = population(rs, lam, n, regime), weights(lam, kind, n)
    ref, S = rm.reference(Y, w)
    B = rm.rank_mu_error_bound(Y, w, kernel, S=S)
    emu = rm.rank_mu_emulated(Y, w, kernel)
    # measured: at most 0.93 (ffma, lambda = 1, where the single rounding of w y is all there is) and 0.14 (tc)
    assert rm.worst_ratio(emu, ref, B) <= 1.0, rm.worst_ratio(emu, ref, B)
    err = np.abs(emu - ref).max()
    assert err > 0 and B.max() / err < VACUITY_CAP[kernel], B.max() / err


@pytest.mark.parametrize('regime,least', [('x2^-12', 50.0), ('log_uniform', 50.0), ('x2^18', np.inf)])
@pytest.mark.parametrize('lam,kind', [(37, 'default'), (129, 'active')])
def test_bound_rejects_the_split_without_column_scales(lam, kind, regime, least):
    """The split at absolute magnitude loses ~2^-25 absolute per operand (lo, then hi subnormal) and overflows above
    65504: the tensor-core bound must reject it by a wide margin (measured 64..260 for small columns, inf for large)."""
    rs = np.random.RandomState(lam * 7 + len(regime))
    Y, w = population(rs, lam, 160, regime), weights(lam, kind)
    ref, S = rm.reference(Y, w)
    B = rm.rank_mu_error_bound(Y, w, 'tc', S=S)
    assert rm.worst_ratio(rm.rank_mu_emulated(Y, w, 'tc_unscaled'), ref, B) >= least
    assert rm.worst_ratio(rm.rank_mu_emulated(Y, w, 'tc'), ref, B) <= 1.0


@pytest.mark.parametrize('kernel', ('ffma', 'tc'))
def test_one_wrong_entry_trips_the_check(kernel):
    rs = np.random.RandomState(3)
    Y, w = population(rs, 64, 160, 'log_uniform'), weights(64, 'active')
    ref, S = rm.reference(Y, w)
    B = rm.rank_mu_error_bound(Y, w, kernel, S=S)
    emu = rm.rank_mu_emulated(Y, w, kernel)
    assert rm.worst_ratio(emu, ref, B) <= 1.0
    for i, j in [(0, 0), (5, 101), (159, 2)]:
        bad = emu.copy()
        bad[i, j] += 1e-4 * S[i, j]
        assert rm.worst_ratio(bad, ref, B) > 1.0
    bad = emu.copy()
    bad[7, 9] = np.nan
    assert rm.worst_ratio(bad, ref, B) == np.inf


@pytest.mark.parametrize('kernel', ('ffma', 'tc'))
def test_bound_is_scale_covariant(kernel):
    """Column j times 2^s_j scales row and column j of the bound (and of the emulated error) by 2^s_j."""
    rs = np.random.RandomState(11)
    Y, w = population(rs, 70, 96, 'log_uniform'), weights(70, 'active', 96)
    s = rs.randint(-20, 21, 96)
    Ys = np.ldexp(Y, s[None, :])
    outer = s[:, None] + s[None, :]
    B, Bs = rm.rank_mu_error_bound(Y, w, kernel), rm.rank_mu_error_bound(Ys, w, kernel)
    np.testing.assert_allclose(Bs, np.ldexp(B, outer), rtol=1e-13, atol=0)
    if kernel == 'tc':
        z, zs = rm.tc_operand(Y, w), rm.tc_operand(Ys, w)
        assert np.array_equal(zs, np.ldexp(z, s[None, :]))
        assert np.array_equal(rm.column_exponents(zs), rm.column_exponents(z) + s)
        assert np.array_equal(rm.rank_mu_emulated(Ys, w, 'tc'), np.ldexp(rm.rank_mu_emulated(Y, w, 'tc'), outer))


def test_column_exponents_put_each_maximum_below_fp16_range():
    z = np.array([[0.0, 1.0, -3.0e4, np.inf, np.nan, 2.0 ** -140, 65504.0 * 4, 0.75],
                  [0.0, -0.5, 1.0, 1.0, 1.0, 0.0, 1.0, -0.25]], np.float32)
    e = rm.column_exponents(z)
    assert e[0] == 0 and e[3] == 0 and e[4] == 0                    # zero and non-finite columns keep their scale
    m = np.ldexp(np.max(np.abs(z[:, [1, 2, 5, 6, 7]]), axis=0).astype(np.float64), -e[[1, 2, 5, 6, 7]])
    assert np.all((m >= 2.0 ** 14) & (m < 2.0 ** 15)), m
    assert np.array_equal(rm.column_exponents(z, scaled=False), np.zeros(8))


def test_tc_halves_follow_the_syrk():
    """k_stages = ceil(lambda / 64) stages of 12 wgmma; the first accumulator takes ceil(k_stages / 2) of them."""
    assert rm.tc_halves(1) == (64, (12, 0))
    assert rm.tc_halves(64) == (64, (12, 0))
    assert rm.tc_halves(65) == (64, (12, 12))
    assert rm.tc_halves(129) == (128, (24, 12))                     # odd k_stages: unequal halves
    assert rm.tc_halves(4096) == (2048, (384, 384))


def test_cov_blend_bound_covers_the_fp32_blend():
    """A numpy stand-in for cma_cov_apply_kernel (fp32 constants, fl(decay C), fl(c1 pc_i), two FMAs emulated with an
    exact fp64 product) stays within the blend bound; an extra error of 8 fp32 roundings of the result does not."""
    rs = np.random.RandomState(5)
    n = 200
    C = (np.eye(n) + 0.01 * rs.randn(n, n)).astype(np.float32)
    dC = rs.randn(n, n).astype(np.float32)
    pc = rs.randn(n).astype(np.float32)
    k = cma.cma_constants(4481, 64)
    c1, cmu = k['c1'], k['cmu']
    decay = 1 - c1 - cmu * k['w'].sum()
    f32 = np.float32
    v = (f32(decay) * C).astype(np.float32)
    v = (v.astype(np.float64) + np.outer((f32(c1) * pc).astype(np.float64), pc)).astype(np.float32)
    got = (v.astype(np.float64) + float(f32(cmu)) * dC.astype(np.float64)).astype(np.float32)
    ref, T = rm.cov_blend_reference(C, dC, pc, decay, c1, cmu)
    B = rm.cov_blend_bound(T)
    assert rm.worst_ratio(got, ref, B) <= 1.0
    assert rm.worst_ratio(got + 8 * rm.U_F32 * np.abs(ref), ref, B) > 1.0
