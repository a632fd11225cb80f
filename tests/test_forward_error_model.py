"""The error model behind tests/test_gpu_forward_error.py, checked on the CPU.

oracle/forward_error.py bounds |a_kernel - a_exact| per action for each des_nes_eval precision; the GPU tests use
that bound, scaled by a measured kappa, as their tolerance.  Here: the bound holds for an emulation of the kernel's
operand rounding and is not vacuous, the GPU case table reaches every eval_tc_kernel instantiation, and the
per-action probe arithmetic recovers injected action errors from fitness values alone.
"""
import numpy as np
import pytest

from oracle import forward_error as fe
from oracle import nes_oracle as orc

SHAPES = [  # d0, H, A, T
    (24, 64, 4, 128),
    (1, 64, 1, 128),
    (3, 128, 8, 128),
    (17, 128, 5, 128),
    (32, 256, 8, 128),
    (31, 256, 7, 128),
]

# max(bound) / max(emulated error) over SHAPES, 2 members each: f16 157..607, f16x3 825..5778, fp32 754..5245.
# The bound adds worst cases over K = H terms per layer where the real errors partly cancel (~sqrt(K)), so the
# factor grows with H; the caps catch a bound that has stopped tracking the error at all.
VACUITY_CAP = {'fp32': 1e4, 'f16': 1e3, 'f16x3': 1e4}


def _member(d0, H, A, T, sigma=0.1):
    obs, _ = orc.synthetic_tape(T, d0, A)
    theta = orc.synthetic_theta(d0, H, A)
    eps = orc.noise(7, 1, 0, 2, orc.param_count(d0, H, A))
    return orc.perturb(theta[None], sigma, eps), obs


@pytest.mark.parametrize('precision', fe.PRECISIONS)
@pytest.mark.parametrize('d0,H,A,T', SHAPES)
def test_emulated_error_within_bound_and_bound_not_vacuous(d0, H, A, T, precision):
    flat, obs = _member(d0, H, A, T)
    ref = orc.forward(flat, obs, d0, H, A)
    B = fe.forward_error_bound(flat, obs, d0, H, A, precision)
    assert B.shape == ref.shape and np.all(B > 0)
    if precision == 'fp32':
        emu = orc.forward(flat, obs, d0, H, A, dtype=np.float32)      # fp32 all through, as the FFMA kernel
    else:
        emu = fe.forward_emulated(flat, obs, d0, H, A, precision)
    err = np.abs(emu - ref)
    assert np.all(err <= B), np.max(err / B)
    assert B.max() / err.max() < VACUITY_CAP[precision], B.max() / err.max()


def test_emulation_rounds_like_the_kernel():
    """f16x3 must be markedly closer to fp64 than f16 (hi/lo split ~2^-22 vs 2^-11), and both nonzero."""
    flat, obs = _member(24, 128, 4, 128)
    ref = orc.forward(flat, obs, 24, 128, 4)
    e16 = np.abs(fe.forward_emulated(flat, obs, 24, 128, 4, 'f16') - ref).max()
    e3 = np.abs(fe.forward_emulated(flat, obs, 24, 128, 4, 'f16x3') - ref).max()
    assert 0 < e3 < e16 / 300, (e3, e16)


def test_weight_error_widens_the_bound():
    flat, obs = _member(24, 64, 4, 128)
    b0 = fe.forward_error_bound(flat, obs, 24, 64, 4, 'f16x3')
    b1 = fe.forward_error_bound(flat, obs, 24, 64, 4, 'f16x3', dtheta=1e-6)
    assert np.all(b1 > b0)


def test_forward_cases_cover_every_tc_instantiation():
    """eval_tc_kernel<H, X3, CL, NA>: H in {64,128,256} x f16/f16x3 x 1-/2-CTA cluster x NA in {4,8} = 24, each with
    one pass and with several; d0 and A cover the W1 paths and unused NA = 8 action rows."""
    seen, passes = set(), {}
    for d0, H, A, T in fe.FORWARD_CASES:
        assert 1 <= d0 <= 32 and 1 <= A <= 8 and T % 128 == 0
        for p in ('f16', 'f16x3'):
            inst = fe.tc_instantiation(H, A, T, p)
            seen.add(inst)
            passes.setdefault(inst, set()).add(fe.tc_passes(T) > 1)
    every = {(H, x3, cl, na) for H in (64, 128, 256) for x3 in (False, True) for cl in (1, 2) for na in (4, 8)}
    assert seen == every
    assert all(v == {False, True} for v in passes.values())
    d0s = {d0 for d0, _, _, _ in fe.FORWARD_CASES}
    assert {1, 3, 16, 17, 24, 31, 32} <= d0s
    assert {d0 % 4 == 0 for d0 in d0s} == {True, False}
    assert {A for _, _, A, _ in fe.FORWARD_CASES} == {1, 2, 4, 5, 7, 8}


def test_tc_instantiation_follows_dispatch_rule():
    assert fe.tc_instantiation(64, 4, 128, 'f16') == (64, False, 1, 4)
    assert fe.tc_instantiation(64, 5, 256, 'f16x3') == (64, True, 2, 8)
    assert fe.tc_instantiation(256, 8, 384, 'f16') == (256, False, 1, 8)
    assert fe.tc_instantiation(128, 1, 512, 'f16x3') == (128, True, 2, 4)
    assert [fe.tc_passes(T) for T in (128, 256, 384, 512)] == [1, 1, 3, 2]


def _stand_in_fitness(actions, target, chunk):
    """A numpy stand-in for the kernel's fitness: fp32 residuals, squared and summed in fp32 per chunk of entries
    (one thread's chain), chunk sums added in fp64, the total rounded to fp32."""
    d = (np.asarray(actions, np.float32) - np.asarray(target, np.float32)).reshape(-1)
    sq = (d * d).astype(np.float32)
    parts = [np.cumsum(sq[i:i + chunk], dtype=np.float32)[-1] for i in range(0, sq.size, chunk)]
    return np.float32(-np.sum(np.asarray(parts, np.float64)))


@pytest.mark.parametrize('T,A,scale', [(128, 4, 1e-7), (128, 8, 1e-3), (512, 7, 3e-7), (256, 1, 0.0)])
def test_probe_recovers_injected_action_errors(T, A, scale):
    rs = np.random.RandomState(T + A)
    exact = np.tanh(rs.randn(T, A))
    target = exact.astype(np.float32)
    inj = scale * rs.randn(T, A)
    inj.reshape(-1)[rs.randint(0, T * A)] += 50 * scale                  # one bad action
    kernel_actions = (exact + inj).astype(np.float32)                     # what a faulty kernel would output
    e_true = kernel_actions.astype(np.float64) - target.astype(np.float64)
    entries = fe.probe_entries(T, A)
    assert len(entries) <= max(512, 1024 if T * A <= 1024 else 0) and len(np.unique(entries)) == len(entries)
    if T * A <= 1024:
        assert len(entries) == T * A
    d = fe.probe_offsets(target, entries)
    assert np.all(np.abs(d - fe.PROBE_DELTA) <= 2.0 ** -24)
    f0 = _stand_in_fitness(kernel_actions, target, 16)
    f = np.empty(len(entries))
    for k, r in enumerate(entries):
        t = target.copy().reshape(-1)
        t[r] = np.float32(t[r] + np.float32(d[k]))
        assert float(t[r]) - float(target.reshape(-1)[r]) == d[k]          # the offset is exact
        f[k] = _stand_in_fitness(kernel_actions, t.reshape(T, A), 16)
    e = fe.probe_recover(f0, f, d)
    res = fe.probe_resolution(d, f0, f, 16)
    got = np.abs(e - e_true.reshape(-1)[entries])
    assert np.all(got <= res), np.max(got / res)
    # the resolution is far below the f16x3 action error (~1e-7)
    if scale <= 3e-7:
        assert np.max(res) < 2e-8


def test_probe_entries_hit_tile_boundaries():
    ent = fe.probe_entries(512, 4)
    rows = set((ent // 4).tolist())
    assert {0, 7, 8, 15, 16, 63, 64, 127, 128, 255, 256, 383, 384, 511} <= rows
    assert len(ent) == 512
    assert np.array_equal(ent, fe.probe_entries(512, 4))                 # fixed sample
