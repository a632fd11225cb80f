"""The reductions of an NES generation entry by entry against fp64: the gradient partial (des_update.cu), the Adam step
and the observation statistics (des_obs.cu).

Gradient.  Thread q of slice c keeps an fp32 FMA chain over the L members of its slice (L = grad_plan's per_chunk, pairs
for the mirrored form), the slices are added in fp64 and the sum is stored as fp32.  The reference is the fp64 sum
ref_j = sum_i s_i eps_ij over the device's own normals (ops.noise_fill), on the GPU in member chunks, and
S_j = sum_i |s_i eps_ij|.  With u = 2^-24, to first order:

    * term i of the kernel is fl(nr s_i) c where noise_fill's eps_ij is fl(nr c): 2u |s_i eps_ij| apart (3u for the
      mirrored form, whose s is fl(s_2i - s_2i+1));
    * the chain of L FMAs rounds L times, each at most u times the partial sum, so at most L u S_j;
    * the fp64 sum of the slices is exact to 2^-53 per slice, and the store rounds once more, by u |g_j|.

So |g_j - ref_j| <= (L + 3) u S_j + u |ref_j|: the rigorous bound has c = 1 (the "+3" also covers the second-order
terms, L u <= 2^-14).  Rounding errors of the chain are not all of one sign, though: they add like a random walk, about
sqrt(L) steps of u times a partial sum of order sqrt(L) |s eps|, and the n/L slices add theirs the same way, so the
error is about u sqrt(n L) |s eps| where the bound has (L + 3) u n |s eps|.  The check therefore uses

    |g_j - ref_j| <= c (L + 3) u S_j + u |ref_j|,   c = min(1, K_GRAD / sqrt(n L)),

n the terms of the sum (members, or pairs).  K_GRAD is measured: (|g_j - ref_j| - u |ref_j|) / ((L + 3) u S_j) times
sqrt(n L), its largest value per case, over every case of this file (one run on an H100 80GB HBM3, 700 W power limit):

    cases                                                    n          L      largest
    plain, 32 members a slice (cap32-*, p448*, ragged-32,    300-5000   30-32  1.35-2.00
      top-offset, gen-70001, state-gen, cancel, runs, sweep)
    plain, forced-1024 / ragged-187                          65536      1024 / 187   1.84 / 1.50
    mirrored pairs-512 / top-offset                          32768 / 2048   512 / 16   2.30 / 1.70
    p5, mirrored-p5, p1 (below u |ref|)                      3-64       3-32   0.007-0.15

so the model holds from n L = 9 to 6.7e7, and K_GRAD = 10 is the largest, 2.30, times 4 rounded up.  Against the old
max|g - ref| <= 1e-5 max|ref| bar that is about 1/3 of it at n = 65536, L = 1024, and 1/15 at n = 1000, L = 32, at
every entry rather than only at the largest.

Adam.  nes_apply's fp64 moments against orc.Adam over 200 generations.  Each generation puts at most 6 fp64 roundings of
its terms between the device's m and the reference's (weight decay, where CUDA contracts g - wd g into an FMA; the two
products; the sum) and 10 between the v's (the square adds its own and doubles the weight decay's), and earlier errors
decay by beta: E_t = beta E_t-1 + k 2^-53 (beta |m_t-1| + (1 - beta) |g_t|) bounds |m_dev - m_ref| entry by entry
(measured at most 0.33 of it for m, 0.20 for v).  The step m^/(sqrt(v^) + eps) is plain IEEE fp64 with no product to
contract: from the device's own m and v it is bit-exact, and so is the fp32 update lr32 * fp32(step) made from it.
Against the fp64 reference the update is within two fp32 roundings, the step's and the product's (one at lr = 1:
measured 0.50 of the bound there, 0.98 at lr = 1e-3), plus what E_m and E_v move the step.  theta equals the reference
theta rebuilt with the device's own updates, bit for bit, including entries of 2^20 that an update of 1e-3 leaves alone.

Observation statistics.  des_obs_normalize is IEEE fp32 and equals numpy bit for bit.  The merges compute in fp64 and
store fp32: m and v within one fp32 rounding of the fp64 result (faithful: less than one ulp apart), n exactly the fp32
count.  The totals merge takes v from raw moments, fmax(fma(-m, m, sumsq/n), 0); the reference restates that formula
with the FMA rounded once (exact rational arithmetic).  So a constant column's v is not 0 but the formula's rounding
noise (1.3e-13 from 4096 samples of -1.3f), within its bound 3 (n + 1) 2^-53 sumsq/n.  The reference's own fp32 online
statistics (utils.py:68-73) do not give 0 there either: 2.7e-13 for 1000 samples of -1.3f, 3.4e-13 for 4096.
des_obs_parts_reduce adds members in order and equals a sequential fp64 sum bit for bit.  The closed-loop rollout and
policy_act normalise inside their kernels and expose only raw observations and actions, so the cross-checks compare
actions: for des_obs_normalize's output (no statistics) and for the raw observations (with them), bit for bit.  No
action is near the clip.  tanh_mufu absorbs many one-ulp steps of an input, so each test also counts the actions that
move when every normalised input moves by one ulp: policy_act 101 of 128 (d0 = 3), 424 of 512 (d0 = 24), 838 of 1024
(d0 = 32); the rollout 89 of 1200 (H = 32), 324 of 1200 (H = 64).  A normaliser one ulp off would move dozens of
actions in every test.  The tape has no normaliser of its own: fitness.TapeSource runs des_obs_normalize on it.

The file runs in 13-16 s on an H100 80GB HBM3 (44 tests; 17-21 s wall with Python's start-up): the fp64 references run on the
GPU in member chunks.

Sensitivity (test_gradient_check_trips_*, test_adam_check_trips_on_fp32_rounding): perturbed references fail the
per-entry checks.  Same run:

    reference                                                  per-entry err/bound   old norm checks / 1e-5
    ragged-32 without member 1481 (|s| = 0.5/4999 = 1.0e-4)    6.7                   0.49: passes it
    p4483, entry P - 1 moved by 2^-10 of itself (|ref| 2.9)    136                   9.0
    m rounded to fp32 once, generation 5                       3.7e7 (m check)       -

The dropped member moves no entry by more than 4e-4, under the old 1e-5 max|ref| bar by a factor of 2; the per-entry
check flags it with a margin of 6.7.
"""
from fractions import Fraction

import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import nes_oracle as orc

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
U64 = 2.0 ** -53
K_GRAD = 10.0        # measured 2.30: see the module docstring
TOP = 1 << 32        # member_range_ok(member_offset, n, 32): member_offset + n <= 2^32


def ops():
    from distributedes_b200 import ops as o
    return o


def dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).to(DEV)


def bits(x):
    x = np.ascontiguousarray(x)
    return x.view({4: np.uint32, 8: np.uint64}[x.dtype.itemsize])


# ---------------------------------------------------------------------------------------------------------------------
# gradient partial
# ---------------------------------------------------------------------------------------------------------------------
def grad_plan(n_local, P):
    """(slices, members per slice) of des_update.cu's grad_plan, 128 threads per CTA and 132 SMs."""
    nq = (P + 3) // 4
    bx = (nq + 127) // 128
    want = (132 * 16 * 2 + bx - 1) // bx
    want = max(min(want, (n_local + 31) // 32), (n_local + 1023) // 1024, 1)
    want = min(want, 65535)
    per_chunk = (n_local + want - 1) // want
    return max((n_local + per_chunk - 1) // per_chunk, 1), per_chunk


def slice_len(n_local, P, mirrored=False):
    """L: the chain length of one thread.  A mirrored shard keeps the plain plan's slices at half as many pairs."""
    per_chunk = grad_plan(n_local, P)[1]
    return (per_chunk + 1) // 2 if mirrored else per_chunk


def grad_reference(shaped, P, seed, gen, member_offset, mirrored=False, chunk=2048):
    """(ref, S) fp64 [P] on the device: sum_i s_i eps_i and sum_i |s_i eps_i| over ops.noise_fill's normals; the
    mirrored form sums (s_2i - s_2i+1) eps_i over pair i's normal (member_offset / 2 + i)."""
    s = shaped.double()
    if mirrored:
        s, member_offset = s[0::2] - s[1::2], member_offset // 2
    ref = torch.zeros(P, dtype=torch.float64, device=DEV)
    S = torch.zeros(P, dtype=torch.float64, device=DEV)
    for o in range(0, s.numel(), chunk):
        k = min(chunk, s.numel() - o)
        eps = ops().noise_fill(k, P, seed, gen, member_offset=member_offset + o, device=DEV).double()
        ref += s[o:o + k] @ eps
        S += s[o:o + k].abs() @ eps.abs_()
    return ref, S


def grad_bound(ref, S, n, L):
    c = min(1.0, K_GRAD / np.sqrt(n * L))
    return c * (L + 3) * U * S + U * ref.abs()


def grad_ratio(g, ref, S, n, L):
    """max_j (|g_j - ref_j| - u |ref_j|) / ((L + 3) u S_j) * sqrt(n L): the quantity K_GRAD bounds."""
    d = (g.double() - ref).abs() - U * ref.abs()
    return float((d / ((L + 3) * U * S).clamp_min(1e-300)).max()) * np.sqrt(n * L)


def check_grad(tag, g, ref, S, n, L):
    d = (g.double() - ref).abs()
    B = grad_bound(ref, S, n, L)
    print('\nGRAD %s n %d L %d  K %.4g  max|d|/B %.3g' % (tag, n, L, grad_ratio(g, ref, S, n, L), float((d / B).max())))
    assert bool((d <= B).all()), (tag, float((d / B).max()))


def shaped_vector(kind, n, P=None, seed=None, gen=None, member_offset=0):
    """fp32 shaped fitness on the device: 'ranks' (centered ranks of random fitness), 'ns' (ns_shape's NSR-ES blend at
    w = 0.5), 'cancel' (pairs s_2k = eps_2k+1,j0 / 4, s_2k+1 = -eps_2k,j0 / 4: column j0 = P - 1 sums to 0 exactly)."""
    rs = np.random.RandomState(n + 7)
    if kind == 'ranks':
        return ops().centered_rank(dev(rs.randn(n)))
    if kind == 'ns':
        return ops().ns_shape(dev(rs.randn(n)), dev(rs.rand(n)), 0.5)
    assert kind == 'cancel' and n % 2 == 0
    e = ops().noise_fill(n, P, seed, gen, member_offset=member_offset, device=DEV)[:, P - 1]
    s = torch.empty_like(e)
    s[0::2], s[1::2] = e[1::2] * 0.25, -e[0::2] * 0.25
    return s


# id: (n_local, P, member_offset, generation, shaped kind, generation through des_state)
GRAD_CASES = {
    'cap32-p73220': (300, 73220, 5000, 11, 'ranks', False),       # 10 slices of 30: at most 32 members a slice
    'cap32-p4481': (1000, 4481, 0, 11, 'ranks', False),           # 32 slices of 32
    'forced-1024': (65536, 73220, 0, 3, 'ranks', False),          # 64 slices of 1024: the slice-length cap
    'ragged-187': (65536, 6020, 0, 3, 'ns', False),               # 351 slices of 187, the last one 86
    'ragged-32': (5000, 6020, 17, 5, 'ranks', False),             # 157 slices of 32, the last one 8
    'p4480': (777, 4480, 1, 2, 'ranks', False),                   # P % 4 = 0 .. 3
    'p4481': (777, 4481, 1, 2, 'ns', False),
    'p4482': (777, 4482, 1, 2, 'ranks', False),
    'p4483': (777, 4483, 1, 2, 'ranks', False),
    'p1': (64, 1, 0, 0, 'ranks', False),
    'p5': (3, 5, 3, 1, 'ranks', False),
    'top-offset': (2048, 6021, TOP - 2048, 9, 'ranks', False),    # the last members a 32-bit counter word addresses
    'gen-70001': (1024, 6022, 100, 70001, 'ns', False),           # a generation word past 2^16
    'state-gen': (1024, 6022, 100, (1 << 32) + 70001, 'ranks', True),   # des_state's 64-bit generation, low word used
    'cancel': (4096, 6023, 0, 4, 'cancel', False),
}
SEED = 0x9E3779B97F4A7C15


def run_grad_case(name):
    n, P, off, gen, kind, via_state = GRAD_CASES[name]
    s = shaped_vector(kind, n, P, SEED, gen, off)
    if via_state:
        g = ops().nes_grad_partial(s, P, seed=SEED, generation=0, state=ops().new_state(DEV, gen), member_offset=off)
    else:
        g = ops().nes_grad_partial(s, P, seed=SEED, generation=gen, member_offset=off)
    ref, S = grad_reference(s, P, SEED, gen, off)
    return s, g, ref, S, n, slice_len(n, P)


@pytest.mark.parametrize('name', list(GRAD_CASES))
def test_gradient_partial_entry_by_entry(name):
    s, g, ref, S, n, L = run_grad_case(name)
    check_grad(name, g, ref, S, n, L)
    if name == 'cancel':       # the cancelled column is tiny against its S, and still within the bound
        assert float(ref[-1].abs()) <= 1e-12 * float(S[-1])


# id: (members, P, member_offset): L = 512 pairs, a ragged plan, and the last pairs of the 32-bit counter
MIRRORED = {'pairs-512': (65536, 73220, 0), 'top-offset': (4096, 6021, TOP - 4096), 'p5': (64, 5, 0)}


@pytest.mark.parametrize('name', list(MIRRORED))
def test_mirrored_pair_form_entry_by_entry(name):
    n, P, off = MIRRORED[name]
    s = shaped_vector('ranks', n)
    g = ops().nes_grad_partial_mirrored(s, P, seed=SEED, generation=6, member_offset=off)
    ref, S = grad_reference(s, P, SEED, 6, off, mirrored=True)
    check_grad('mirrored-' + name, g, ref, S, n // 2, slice_len(n, P, mirrored=True))


def test_runs_and_sweep_partials_entry_by_entry():
    """nes_grad_partial_runs (run r at member_offset r N) and nes_grad_partial_sweep (run r under its own seed at
    member_offset 0), every run against its own fp64 reference."""
    from distributedes_b200 import ops_runs, ops_sweep
    R, N, P, gen = 3, 1500, 4483, 8
    rs = np.random.RandomState(4)
    shaped = torch.stack([ops().centered_rank(dev(rs.randn(N))) for _ in range(R)]).contiguous()
    L = slice_len(N, P)
    g = ops_runs.nes_grad_partial_runs(shaped, P, seed=SEED, generation=gen)
    for r in range(R):
        ref, S = grad_reference(shaped[r], P, SEED, gen, r * N)
        check_grad('runs-%d' % r, g[r], ref, S, N, L)
    seeds = [5, (1 << 40) + 7, 123456789]
    hp = ops_sweep.run_table(seeds, [0.1, 0.05, 0.2], 0.01, 0.005, 0.0, DEV)
    g = ops_sweep.nes_grad_partial_sweep(shaped, P, hp, generation=gen)
    for r in range(R):
        ref, S = grad_reference(shaped[r], P, seeds[r], gen, 0)
        check_grad('sweep-%d' % r, g[r], ref, S, N, L)


def _old_check(g, ref):
    """The norm checks of test_gpu_ops.py: the larger of the two ratios over its 1e-5 bar (<= 1 passes)."""
    d = g.double() - ref
    return max(float(d.norm() / ref.norm()), float(d.abs().max() / ref.abs().max())) / 1e-5


def _new_check(g, ref, S, n, L):
    return float(((g.double() - ref).abs() / grad_bound(ref, S, n, L)).max())


def test_gradient_check_trips_on_a_dropped_member():
    """The fp64 reference without one member of one slice (the member with the smallest nonzero |s|, 0.5/4999) fails
    the per-entry check."""
    s, g, ref, S, n, L = run_grad_case('ragged-32')
    _, _, off, gen, _, _ = GRAD_CASES['ragged-32']
    a = s.double().abs()
    i = int(torch.where(a > 0, a, torch.full_like(a, np.inf)).argmin())
    eps = ops().noise_fill(1, g.numel(), SEED, gen, member_offset=off + i, device=DEV).double()[0]
    dropped = ref - float(s[i]) * eps
    new, old = _new_check(g, dropped, S, n, L), _old_check(g, dropped)
    print('\nSENSITIVITY dropped member %d (|s| %.3g): per-entry %.3g, old norm check %.3g'
          % (i, abs(float(s[i])), new, old))
    assert _new_check(g, ref, S, n, L) <= 1 and new > 1
    assert old <= 1                     # the norm checks of test_gpu_ops.py would have passed it


def test_gradient_check_trips_on_a_moved_tail_entry():
    """Entry P - 1 (the last, partial quad) of the fp64 reference moved by 2^-10 of its own magnitude fails the
    per-entry check."""
    s, g, ref, S, n, L = run_grad_case('p4483')
    moved = ref.clone()
    moved[-1] *= 1 + 2.0 ** -10
    new, old = _new_check(g, moved, S, n, L), _old_check(g, moved)
    print('\nSENSITIVITY tail entry |ref| %.3g (max %.3g): per-entry %.3g, old norm check %.3g' %
          (float(ref[-1].abs()), float(ref.abs().max()), new, old))
    assert new > 1


# ---------------------------------------------------------------------------------------------------------------------
# Adam
# ---------------------------------------------------------------------------------------------------------------------
class AdamRun:
    """One run's fp64 reference (orc.Adam through orc.nes_update) beside the device's apply, checked every generation:
    returns the largest ratio of each error to its bound (<= 1 passes)."""

    def __init__(self, theta0, N, sigma, lr, wd, beta1=0.9, beta2=0.999, eps=1e-8, round_m_at=None):
        P = theta0.size
        self.opt = orc.Adam(beta1, beta2, eps)
        self.opt.m, self.opt.v = np.zeros(P), np.zeros(P)
        self.N, self.sigma, self.lr, self.wd = N, sigma, lr, wd
        self.Em, self.Ev = np.zeros(P), np.zeros(P)
        self.theta = theta0.copy()
        self.t, self.round_m_at = 0, round_m_at

    def step(self, partial, g_dev, m_dev, v_dev, upd_dev, theta_dev):
        o, b1, b2 = self.opt, self.opt.beta1, self.opt.beta2
        g = partial.astype(np.float64) / self.N / self.sigma                  # natural_es.py:92, as apply_at
        assert np.array_equal(bits(g_dev), bits(g))
        gw = g - self.wd * g
        m0, v0 = o.m.copy(), o.v.copy()
        _, upd_ref = orc.nes_update(self.theta, g, o, self.wd, self.lr)
        if self.round_m_at == self.t:           # sensitivity: one step's m through fp32
            o.m = o.m.astype(np.float32).astype(np.float64)
        self.t += 1
        self.Em = b1 * self.Em + 6 * U64 * (b1 * np.abs(m0) + (1 - b1) * np.abs(gw))
        self.Ev = b2 * self.Ev + 10 * U64 * (b2 * v0 + (1 - b2) * gw * gw)
        r_m = np.max(np.abs(m_dev - o.m) / np.maximum(self.Em, 1e-300), initial=0, where=self.Em > 0)
        r_v = np.max(np.abs(v_dev - o.v) / np.maximum(self.Ev, 1e-300), initial=0, where=self.Ev > 0)
        exact_mv = np.array_equal(m_dev[self.Em == 0], o.m[self.Em == 0]) and np.array_equal(v_dev[self.Ev == 0],
                                                                                               o.v[self.Ev == 0])
        # the step from the device's own moments: bit-exact, and so is the fp32 update
        c1, c2 = 1.0 - o.beta1_t, 1.0 - o.beta2_t
        step_dev = (m_dev / c1) / (np.sqrt(v_dev / c2) + o.epsilon)
        lr32 = np.float32(self.lr)
        same_update = np.array_equal(bits(upd_dev), bits((lr32 * step_dev.astype(np.float32)).astype(np.float32)))
        # against the fp64 step: two fp32 roundings, plus what E_m and E_v move the step
        vh = o.v / c2
        step = (o.m / c1) / (np.sqrt(vh) + o.epsilon)
        dstep = (self.Em / c1) / (np.sqrt(vh) + o.epsilon) + 0.5 * np.abs(step) * np.divide(
            self.Ev, o.v, out=np.zeros_like(self.Ev), where=o.v > 0) + 8 * U64 * np.abs(step)
        ref64 = float(lr32) * step
        bound = (2 * U + U * U) * np.abs(ref64) + float(lr32) * dstep * (1 + 3 * U)
        r_u = np.max(np.abs(upd_dev - ref64) / np.maximum(bound, 1e-300), initial=0, where=bound > 0)
        zero_ok = np.all(upd_dev[bound == 0] == ref64[bound == 0])
        self.theta = (self.theta + upd_dev).astype(np.float32)               # natural_es.py:96 with the device's update
        same_theta = np.array_equal(bits(theta_dev), bits(self.theta))
        return dict(m=r_m, v=r_v, update=r_u, exact=exact_mv and zero_ok and same_update and same_theta,
                    same_update=same_update, same_theta=same_theta)


def adam_partials(rs, P, N, scale, zeros):
    """One generation's partial sums: entry j at its own scale, some entries always 0, 1% 0 this generation."""
    p = rs.randn(P) * scale * N * 0.01
    p[zeros] = 0.0
    p[rs.rand(P) < 0.01] = 0.0
    return p.astype(np.float32)


def adam_setup(P, seed):
    rs = np.random.RandomState(seed)
    scale = 10.0 ** rs.uniform(-5, 2, P)
    zeros = np.arange(0, P, 97)
    theta0 = (rs.randn(P) * 0.1).astype(np.float32)
    theta0[1::211] = np.float32(2.0 ** 20)                 # updates below half its ulp round away
    theta0[2::211] = np.float32(-3.0e-5)
    return rs, scale, zeros, theta0


def _summarise(tag, worst):
    print('\nADAM %s max m err/bound %.3g, v %.3g, update %.3g' % (tag, worst['m'], worst['v'], worst['update']))


@pytest.mark.parametrize('lr,wd', [(1e-3, 0.0), (1e-3, 0.005), (1.0, 0.0), (1.0, 0.005)])
def test_adam_200_generations_entry_by_entry(lr, wd):
    o = ops()
    P, N, sigma, G = 6020, 4096, 0.1, 200
    rs, scale, zeros, theta0 = adam_setup(P, 3)
    theta = dev(theta0)
    m = torch.zeros(P, dtype=torch.float64, device=DEV)
    v = torch.zeros(P, dtype=torch.float64, device=DEV)
    upd = torch.empty(P, dtype=torch.float32, device=DEV)
    g64 = torch.empty(P, dtype=torch.float64, device=DEV)
    st = o.new_state(DEV, generation=12)
    ref = AdamRun(theta0, N, sigma, lr, wd)
    worst = dict(m=0.0, v=0.0, update=0.0)
    for t in range(G):
        partial = adam_partials(rs, P, N, scale, zeros)
        o.nes_apply(theta, m, v, dev(partial), N, st, sigma=sigma, learning_rate=lr, weight_decay=wd, update_out=upd,
                    grad_out=g64)
        o.state_advance(st)
        r = ref.step(partial, g64.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(), upd.cpu().numpy(),
                     theta.cpu().numpy())
        assert r['exact'] and r['m'] <= 1 and r['v'] <= 1 and r['update'] <= 1, (t, r)
        worst = {k: max(worst[k], r[k]) for k in worst}
    _summarise('lr %g wd %g' % (lr, wd), worst)
    # beta^t on the device: the same product of 200 factors as Adam's beta_t *= beta, and 0.9^200 to its rounding
    s = o.read_state(st)
    assert s['generation'] == 12 + G and s['adam_t'] == G
    assert s['beta1_t'] == ref.opt.beta1_t and s['beta2_t'] == ref.opt.beta2_t
    assert abs(s['beta1_t'] - 0.9 ** G) <= G * U64 * 0.9 ** G and abs(s['beta2_t'] - 0.999 ** G) <= G * U64 * 0.999 ** G
    th = theta.cpu().numpy()
    assert not np.array_equal(th, theta0)
    if lr == 1e-3:                              # |update| < 2^-4, half an ulp of 2^20: those entries never move
        assert np.array_equal(th[1::211], theta0[1::211])


@pytest.mark.parametrize('kind', ['runs', 'sweep'])
def test_adam_runs_and_sweep_entry_by_entry(kind):
    """nes_apply_runs (one optimiser for every run) and nes_apply_sweep (sigma, learning rate and weight decay per run)
    over 200 generations, every run against its own fp64 reference; the runs share one des_state."""
    from distributedes_b200 import ops_runs, ops_sweep
    o = ops()
    R, P, N, G = 3, 1000, 64, 200
    hps = [(0.1, 1e-3, 0.0), (0.02, 1.0, 0.005), (0.5, 0.05, 0.005)] if kind == 'sweep' else [(0.05, 0.3, 0.005)] * R
    rs, scale, zeros, theta0 = adam_setup(R * P, 5)
    theta0 = theta0.reshape(R, P)
    theta = dev(theta0)
    m = torch.zeros((R, P), dtype=torch.float64, device=DEV)
    v = torch.zeros((R, P), dtype=torch.float64, device=DEV)
    upd = torch.empty((R, P), dtype=torch.float32, device=DEV)
    g64 = torch.empty((R, P), dtype=torch.float64, device=DEV)
    st = o.new_state(DEV)
    refs = [AdamRun(theta0[r], N, *hps[r]) for r in range(R)]
    hp = ops_sweep.run_table([1, 2, 3], [h[0] for h in hps], [h[1] for h in hps], [h[2] for h in hps], 0.0, DEV)
    worst = dict(m=0.0, v=0.0, update=0.0)
    for t in range(G):
        partial = adam_partials(rs, R * P, N, scale, zeros).reshape(R, P)
        if kind == 'sweep':
            ops_sweep.nes_apply_sweep(theta, m, v, dev(partial), N, st, hp, update_out=upd, grad_out=g64)
        else:
            sigma, lr, wd = hps[0]
            ops_runs.nes_apply_runs(theta, m, v, dev(partial), N, st, sigma=sigma, learning_rate=lr, weight_decay=wd,
                                    update_out=upd, grad_out=g64)
        o.state_advance(st)
        got = [x.cpu().numpy() for x in (g64, m, v, upd, theta)]
        for r in range(R):
            res = refs[r].step(partial[r], *(x[r] for x in got))
            assert res['exact'] and res['m'] <= 1 and res['v'] <= 1 and res['update'] <= 1, (t, r, res)
            worst = {k: max(worst[k], res[k]) for k in worst}
    _summarise(kind, worst)


def test_adam_check_trips_on_fp32_rounding():
    """The reference's m rounded to fp32 once, at generation 5, where Adam keeps it in fp64: the m check fails there."""
    o = ops()
    P, N = 6020, 4096
    rs, scale, zeros, theta0 = adam_setup(P, 3)
    theta = dev(theta0)
    m = torch.zeros(P, dtype=torch.float64, device=DEV)
    v = torch.zeros(P, dtype=torch.float64, device=DEV)
    upd = torch.empty(P, dtype=torch.float32, device=DEV)
    g64 = torch.empty(P, dtype=torch.float64, device=DEV)
    st = o.new_state(DEV)
    ref = AdamRun(theta0, N, 0.1, 0.01, 0.005, round_m_at=5)
    ratios = []
    for t in range(6):
        partial = adam_partials(rs, P, N, scale, zeros)
        o.nes_apply(theta, m, v, dev(partial), N, st, sigma=0.1, learning_rate=0.01, weight_decay=0.005,
                    update_out=upd, grad_out=g64)
        o.state_advance(st)
        ratios.append(ref.step(partial, g64.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(), upd.cpu().numpy(),
                               theta.cpu().numpy())['m'])
    print('\nSENSITIVITY adam m rounded to fp32 at generation 5: m err/bound %s' % ['%.3g' % r for r in ratios])
    assert max(ratios[:5]) <= 1 and ratios[5] > 1


# ---------------------------------------------------------------------------------------------------------------------
# observation statistics
# ---------------------------------------------------------------------------------------------------------------------
def np_normalize(obs, m, v):
    """utils.py:50-51 in numpy fp32: (o - m) / sqrt(v + 1e-6)."""
    return (obs - m) / np.sqrt(v + np.float32(1e-6))


def stats_vector(m, v, n):
    return np.concatenate([m, v, [n]]).astype(np.float32)


@pytest.mark.parametrize('T,d0', [(7, 1), (33, 3), (100, 24), (3, 1024), (1, 3), (257, 5)])
def test_obs_normalize_bit_for_bit(T, d0):
    rs = np.random.RandomState(T * d0)
    obs = (rs.randn(T, d0) * 10.0 ** rs.uniform(-3, 3, d0)).astype(np.float32)
    m = (rs.randn(d0) * 3).astype(np.float32)
    v = (np.abs(rs.randn(d0)) * 10.0 ** rs.uniform(-8, 4, d0)).astype(np.float32)
    v[::3] = 0.0                                           # v = 0: sqrt(1e-6)
    st = stats_vector(m, v, 1234.0)
    got = ops().obs_normalize(dev(obs), dev(st)).cpu().numpy()
    assert np.array_equal(bits(got), bits(np_normalize(obs, m, v)))
    empty = stats_vector(m, v, 0.0)                        # n = 0: the observations pass through
    assert np.array_equal(bits(ops().obs_normalize(dev(obs), dev(empty)).cpu().numpy()), bits(obs))


def faithful(got, ref):
    """got is one of the two fp32 neighbours of the fp64 ref: |got - ref| < ulp at |ref|."""
    ref = np.asarray(ref, np.float64)
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    return np.abs(np.asarray(got, np.float64) - ref) <= ulp


def chan64(mA, vA, nA, mb, vb, nB):
    n = nA + nB
    delta = mb - mA
    return mA + delta * nB / n, (vA * nA + vb * nB + delta * delta * nA * nB / n) / n, n


def test_obs_stats_merge_tape():
    """des_obs_stats_merge: the first merge, four repeated merges (each from the device's own statistics), a column at
    offset 1e4 with spread 1e-2, d0 = 24 and 1024."""
    for d0, T in ((24, 200), (1024, 37)):
        rs = np.random.RandomState(d0)
        st = torch.zeros(2 * d0 + 1, dtype=torch.float32, device=DEV)
        for k, n_feed in enumerate([T * 64, T * 64 * 10, 3.0e6, 1.0, 777.0 * T]):
            obs = (rs.randn(T, d0) * 2 + k).astype(np.float32)
            obs[:, 1] = (1.0e4 + 1.0e-2 * rs.randn(T)).astype(np.float32)
            A = st.cpu().numpy().astype(np.float64)
            o64 = obs.astype(np.float64)
            mb = o64.mean(0)
            vb = ((o64 - mb) ** 2).mean(0)
            m, v, n = chan64(A[:d0], A[d0:2 * d0], A[2 * d0], mb, vb, float(n_feed))
            ops().obs_stats_merge(st, dev(obs), n_feed)
            got = st.cpu().numpy()
            assert faithful(got[:d0], m).all() and faithful(got[d0:2 * d0], v).all(), (d0, k)
            assert got[2 * d0] == np.float32(n), (d0, k)


def test_obs_parts_reduce_in_member_order():
    rs = np.random.RandomState(9)
    d0, n = 511, 3001
    w = 2 * d0 + 1
    parts = rs.randn(n, w) * 10.0 ** rs.uniform(-6, 6, (n, 1))
    got = ops().obs_parts_reduce(dev(parts, torch.float64), d0).cpu().numpy()
    assert np.array_equal(bits(got), bits(np.cumsum(parts, axis=0)[-1]))     # sequential fp64, member 0 first


def _totals(obs):
    """[sum | sum of squares | count] of obs[T, d0] as the kernels accumulate them: fp64, in order."""
    o = obs.astype(np.float64)
    return np.concatenate([np.cumsum(o, 0)[-1], np.cumsum(o * o, 0)[-1], [float(len(obs))]])


def _merge_cases(d0, rs):
    """(stats fp32 [2 d0 + 1], totals fp64 [2 d0 + 1], what to check) rows."""
    rows = []
    obs = rs.randn(500, d0).astype(np.float32) * 3 + 1
    rows.append((stats_vector(rs.randn(d0), np.abs(rs.randn(d0)), 40.0), np.zeros(2 * d0 + 1), 'untouched'))
    t = _totals(obs)
    t[2 * d0] = 0.0
    rows.append((stats_vector(rs.randn(d0), np.abs(rs.randn(d0)), 40.0), t, 'untouched'))   # sums without a count
    rows.append((np.zeros(2 * d0 + 1, np.float32), _totals(obs), 'chan'))                   # the first merge
    cst = np.tile(np.float32([0.1, -1.3, 3.0, 0.7071])[np.arange(d0) % 4], (1000, 1))
    rows.append((np.zeros(2 * d0 + 1, np.float32), _totals(cst), 'constant'))
    cst2 = np.tile(np.float32([0.1, -1.3, 3.0, 0.7071])[np.arange(d0) % 4], (4096, 1))
    rows.append((stats_vector(cst2[0], np.zeros(d0), 1000.0), _totals(cst2), 'constant'))  # merged into itself
    rows.append((stats_vector(rs.randn(d0), np.abs(rs.randn(d0)), 2.0 ** 24 - 1), _totals(obs[:4]), 'chan'))
    rows.append((stats_vector(rs.randn(d0) * 0.1, np.abs(rs.randn(d0)), 3.0e7), _totals(obs), 'chan'))
    rows.append((stats_vector(rs.randn(d0) * 50, np.abs(rs.randn(d0)) * 1e-3, 12.0), _totals(obs * 0.01), 'chan'))
    off = (1.0e4 + 1.0e-2 * rs.randn(500, d0)).astype(np.float32)          # large offset, small spread: raw moments
    rows.append((np.zeros(2 * d0 + 1, np.float32), _totals(off), 'chan'))  # cancel, the kernel's formula is pinned
    return rows


def raw_variance(sums, sumsq, nB):
    """The kernels' batch moments from the totals: mb = sum/nB, vb = fmax(fma(-mb, mb, sumsq/nB), 0) with the FMA
    rounded once (exact rational arithmetic, then one rounding to fp64)."""
    mb = sums / nB
    q = sumsq / nB
    vb = np.array([float(Fraction(float(qk)) - Fraction(float(mk)) ** 2) for mk, qk in zip(mb, q)])
    return mb, np.maximum(vb, 0.0), q


def _check_merge(got, stats, totals, what, d0):
    if what == 'untouched':
        return np.array_equal(bits(got), bits(stats))
    nB = totals[2 * d0]
    mb, vb, q = raw_variance(totals[:d0], totals[d0:2 * d0], nB)
    A = stats.astype(np.float64)
    m, v, n = chan64(A[:d0], A[d0:2 * d0], A[2 * d0], mb, vb, nB)
    ok = got[2 * d0] == np.float32(np.float32(A[2 * d0]) + np.float32(nB))       # the fp32 count, rounded past 2^24
    # the Chan sums of nonnegative terms: CUDA's contractions move v by a few fp64 roundings of itself
    vok = np.abs(got[d0:2 * d0] - v) <= np.spacing(np.abs(v).astype(np.float32)) + 4 * U64 * np.abs(v)
    ok = ok and faithful(got[:d0], m).all() and vok.all()
    if what == 'constant':
        # the mean is the constant; v is the raw formula's rounding noise, not 0 (the reference's fp32 online
        # statistics leave noise too: 2.7e-13 for 1000 samples of -1.3f), within its bound 3 (nB + 1) 2^-53 sumsq/nB
        ok = ok and np.array_equal(got[:d0], stats[:d0] if A[2 * d0] else mb.astype(np.float32)) and \
            np.all(got[d0:2 * d0] <= 3 * (nB + 1) * U64 * q)
    return ok


@pytest.mark.parametrize('d0', [3, 24, 1024])
def test_obs_stats_merge_totals_edges(d0):
    """des_obs_stats_merge_totals row by row and des_obs_stats_merge_totals_runs on all rows at once: nB = 0 leaves the
    bytes alone, the first merge, constant columns (their mean exact, v the raw formula's rounding noise), a count
    crossing 2^24 rounds as fp32 nA + nB, a column at offset 1e4 with spread 1e-2, and everything against fp64 Chan on
    the kernel's raw-moment formula within one fp32 rounding."""
    from distributedes_b200 import ops_runs
    rows = _merge_cases(d0, np.random.RandomState(d0))
    for stats, totals, what in rows:
        got = ops().obs_stats_merge_totals(dev(stats), dev(totals, torch.float64), d0).cpu().numpy()
        assert _check_merge(got, stats, totals, what, d0), what
    S = np.stack([r[0] for r in rows])
    T = np.stack([r[1] for r in rows])
    got = ops_runs.obs_stats_merge_totals_runs(dev(S), dev(T, torch.float64), d0).cpu().numpy()
    for r, (stats, totals, what) in enumerate(rows):
        assert _check_merge(got[r], stats, totals, what, d0), (r, what)
    assert float(got[5, 2 * d0]) == 2.0 ** 24 + 4          # 2^24 - 1 + 4 rounds to even, as fp32 nA + nB does


CLIP = 1.0e3            # far above every action below: no clip can hide a difference


def one_ulp_changes(o, rows, x, alive, kw, a):
    """How many actions move when every normalised input moves by one ulp: how visible a normaliser one ulp off is to
    an action comparison.  tanh_mufu absorbs most such steps, so only a share of the actions move."""
    b = o.policy_act(rows, torch.nextafter(x, torch.full_like(x, np.inf)).contiguous(), alive, **kw)
    return int((b != a).sum())


def _stats(d0, rs):
    """(m, v, n) of observations of order 1; column d0 // 2 has v = 0 (sqrt(1e-6) in the normaliser)."""
    m = (rs.randn(d0) * 0.5).astype(np.float32)
    v = (np.abs(rs.randn(d0)) * 10.0 ** rs.uniform(-1, 1, d0)).astype(np.float32)
    v[d0 // 2] = 0.0
    return m, v, 5000.0


@pytest.mark.parametrize('d0,H,A', [(3, 32, 1), (24, 64, 4), (32, 128, 8)])
def test_policy_act_normalises_as_obs_normalize(d0, H, A):
    """policy_act with statistics gives, bit for bit, the actions it gives for des_obs_normalize's output without."""
    o = ops()
    rs = np.random.RandomState(d0)
    n, reps = 8, 16
    P = orc.param_count(d0, H, A)
    rows = dev(np.stack([orc.synthetic_theta(d0, H, A, seed=i) for i in range(n)]))     # nn.Linear-style weights
    m, v, cnt = _stats(d0, rs)
    obs = rs.randn(n, reps, d0) * 2
    obs[..., d0 // 2] = m[d0 // 2] + 1e-3 * rs.randn(n, reps)      # the zero-variance column: at its mean
    obs = dev(obs.astype(np.float32))
    alive = torch.ones((n, reps), dtype=torch.uint8, device=DEV)
    st = dev(stats_vector(m, v, cnt))
    kw = dict(state_dim=d0, hidden=H, action_dim=A, repetitions=reps, clip=CLIP, seed=3, generation=2, t=4)
    a = o.policy_act(rows, obs, alive, obs_stats=st, **kw)
    x = o.obs_normalize(obs.reshape(n * reps, d0), st).reshape(n, reps, d0).contiguous()
    b = o.policy_act(rows, x, alive, **kw)
    assert torch.equal(a, b)
    assert float(a.abs().max()) < CLIP / 10
    moved = one_ulp_changes(o, rows, x, alive, kw, a)
    print('\nNORMALISER policy_act d0 %d: one ulp on every input moves %d of %d actions' % (d0, moved, a.numel()))
    assert moved >= 10


@pytest.mark.parametrize('H', [32, 64])
def test_rollout_normalises_as_obs_normalize(H):
    """The closed-loop rollout's recorded actions at steps 0..59 are policy_act's for the recorded raw observations with
    the same statistics, and for des_obs_normalize's output of them without: all three bit for bit.  The clip is out of
    reach, so the recorded actions are the forward's own."""
    o = ops()
    rs = np.random.RandomState(H)
    n, reps, horizon, off = 2, 10, 60, 6
    P = orc.param_count(3, H, 1)
    rows = dev((orc.synthetic_theta(3, H, 1, seed=H) + 0.2 * rs.randn(n, P)).astype(np.float32))
    st = dev(stats_vector(*_stats(3, rs)))
    obs_rec = torch.empty((n, reps, horizon, 3), dtype=torch.float32, device=DEV)
    act_rec = torch.empty((n, reps, horizon, 1), dtype=torch.float32, device=DEV)
    o.rollout_record_solutions(rows, hidden=H, horizon=horizon, repetitions=reps, clip=CLIP, seed=11, generation=3,
                               member_offset=off, obs_stats=st, obs_out=obs_rec, actions_out=act_rec)
    assert float(act_rec.abs().max()) < CLIP / 10
    alive = torch.ones((n, reps), dtype=torch.uint8, device=DEV)
    kw = dict(state_dim=3, hidden=H, action_dim=1, repetitions=reps, clip=CLIP, seed=11, generation=3,
              member_offset=off)
    moved = []
    for t in range(horizon):
        raw = obs_rec[:, :, t].contiguous()
        a = o.policy_act(rows, raw, alive, obs_stats=st, t=t, **kw)
        x = o.obs_normalize(raw.reshape(n * reps, 3), st).reshape(n, reps, 3).contiguous()
        b = o.policy_act(rows, x, alive, t=t, **kw)
        assert torch.equal(a, act_rec[:, :, t]) and torch.equal(a, b), t
        moved.append(one_ulp_changes(o, rows, x, alive, dict(kw, t=t), a))
    print('\nNORMALISER rollout H %d: one ulp on every input moves %d of %d actions' % (H, sum(moved), act_rec.numel()))
    assert sum(moved) >= 10
