"""des_nes_eval as an error meter: every action of the forward checked against fp64, per eval kernel instantiation.

The fitness is -sum_t ||clip(a_t) - a*_t||^2.  With the GPU's own perturbed weights theta' (ops.nes_perturb), the
target a* = fp32(forward_fp64(theta', obs)) and a clip nothing reaches, the fitness is -sum e^2 with e = a_gpu - a*:
no clipping, no dilution, and |e| <= sqrt(-fitness) for every single action.  Moving one target entry r by d then
recovers e_r itself: f_r = f0 + 2 d e_r - d^2 (per-action probes, oracle/forward_error.py).

Every check also runs on the odd member 2p + 1 of a mirrored pair (des_nes_eval_mirrored, theta' = theta - sigma*eps_p,
the row ops.nes_perturb_mirrored gives): the eval_tc_mirrored_kernel instantiations and the FFMA kernel's mirrored
path, whose producers apply the member's sign at six places of their own.  The even member 2p must give the bits of
plain member p on every case.

Tolerances are kappa * B, B = oracle.forward_error.forward_error_bound (a worst-case bound that never lets errors
cancel).  The bound sits two to four orders of magnitude above the real error, so an unscaled B would wave through
real bugs.  kappa is therefore set from the measured maximum of err/B: one run of every residual case
(FORWARD_CASES x 3 precisions, ||e||_2 / ||B||_2) and every probe case (PROBE_CASES, max_r |e_r| / B_r) of this file on
an H100 SXM (80 GB, 132 SMs; power limit not recorded), rounded up from 4x that maximum:

    precision   residual max   KAPPA_RESIDUAL   probe max   KAPPA_PROBE
    fp32        0.00114        0.005            0.00547     0.022
    f16         0.00420        0.017            0.0141      0.06
    f16x3       0.00108        0.0045           0.00340     0.014

The mirrored odd members, measured the same way in one run on an H100 80GB HBM3 (SXM) at a 700 W power limit and a
1980 MHz max SM clock, driver 580.159.03, in which the plain maxima above came out again digit for digit:

    precision   residual max   probe max
    fp32        0.00114        0.00497
    f16         0.00608        0.0136
    f16x3       0.00131        0.00394

The kernels are deterministic, so these maxima repeat run to run; the 4x covers other compilers and drivers.
The mirrored f16 and f16x3 residual maxima and the f16x3 probe maximum sit above the plain ones (kappa is 2.8x, 3.4x
and 3.6x above them), and kappa is unchanged: nothing in the odd member's arithmetic differs, err/B simply varies from
member to member, and kappa was set from one member per case.  At (1, 64, 1, 128), the shape of both residual maxima,
oracle.forward_error.forward_emulated (the kernel's fp16 operands, fp64 everything else) gives 0.00610 for the odd f16
member measured at 0.00608.  Over members 0..63 at that shape, plain against odd: median 0.00399 / 0.00426 and max
0.00718 / 0.00750 (f16), median 0.00092 / 0.00097 and max 0.00238 / 0.00219 (f16x3).  Probes over members 0..15 at
(3, 64, 7, 128), the shape of every probe maximum: median 0.0138 / 0.0147 (f16), 0.00359 / 0.00356 (f16x3).
What a single wrong action must be to fail the checks (test_checks_trip_on_one_wrong_action) at the headline shape
(24, 256, 4, 256): the probe flags an action off by 2 KAPPA_PROBE B_r = 1.4e-4 (fp32), 0.087 (f16), 1.1e-4 (f16x3)
at the median B_r; the residual assert fails for one action off by 2 KAPPA_RESIDUAL ||B||_2 = 1.0e-3 (fp32),
0.79 (f16), 1.1e-3 (f16x3).
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import forward_error as fe
from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
SEED, GEN, SIGMA = 2024, 3, 0.1
KAPPA_RESIDUAL = {'fp32': 0.005, 'f16': 0.017, 'f16x3': 0.0045}      # measured max 0.00114, 0.00420, 0.00108
KAPPA_PROBE = {'fp32': 0.022, 'f16': 0.06, 'f16x3': 0.014}           # measured max 0.00547, 0.0141, 0.00340
HEADLINE = (24, 256, 4, 256)
GROUPS = ('W1', 'b1', 'W2', 'b2', 'W3', 'b3')                        # orc.unflatten's order


def ops():
    from distributedes_b200 import ops as _ops
    return _ops


def _dtheta(flat, theta, precision):
    """The tensor-core kernel generates theta' as fma(sqrt(sigma^2 ...) cos, theta) instead of nes_perturb's
    fma(sigma, z, theta): the two agree to 2^-20 of sigma*|eps| plus one ulp of theta'.  The odd member of a mirrored
    pair negates the folded radius, fma(-r, c, theta), against nes_perturb_mirrored's fma(-sigma, z, theta): the same
    bound.  The FFMA kernel and nes_perturb share the formula, mirrored or not."""
    if precision == 'fp32':
        return 0.0
    f, t = flat.astype(np.float64), theta.astype(np.float64)
    return 2.0 ** -20 * np.abs(f - t) + 2.0 ** -23 * np.abs(f)


def _group_slices(d0, H, A):
    """Flat index ranges of W1, b1, W2, b2, W3 and b3."""
    sizes = [H * d0, H, H * H, H, A * H, A]
    return {g: slice(int(e - n), int(e)) for g, n, e in zip(GROUPS, sizes, np.cumsum(sizes))}


class Case:
    """One member's residual tape for shape (d0, H, A, T): target = fp32 of the fp64 forward of the GPU's theta'.

    The member is `member` of des_nes_eval; mirrored, it is the odd member 2*member + 1 of des_nes_eval_mirrored,
    theta - sigma*eps with the eps of plain member `member`, evaluated by a launch of its whole pair."""

    def __init__(self, d0, H, A, T, precision, member, sigma=SIGMA, clip=None, obs_seed=None, mirrored=False):
        self.d0, self.H, self.A, self.T, self.precision, self.member, self.sigma = d0, H, A, T, precision, member, sigma
        self.mirrored = mirrored
        obs, _ = orc.synthetic_tape(T, d0, A, seed=obs_seed if obs_seed is not None else 31 * T + d0)
        self.obs = obs
        self.theta = orc.synthetic_theta(d0, H, A, seed=H + A)
        self.th = torch.from_numpy(self.theta).to(DEV)
        self.o = torch.from_numpy(obs).to(DEV)
        if mirrored:
            rows = ops().nes_perturb_mirrored(self.th, 2, sigma, SEED, GEN, member_offset=2 * member)
        else:
            rows = ops().nes_perturb(self.th, 1, sigma, SEED, GEN, member_offset=member)
        self.clip = clip
        self.set_flat(rows.cpu().numpy()[-1])

    def set_flat(self, flat):
        """Reference the case to the weights `flat`: a_ref = forward(flat), its bound B and the target fp32(a_ref).
        The clip, unless given, is one the forward of the first weights never reaches."""
        d0, H, A = self.d0, self.H, self.A
        self.flat = flat
        self.a_ref = orc.forward(flat, self.obs, d0, H, A)
        self.B = fe.forward_error_bound(flat, self.obs, d0, H, A, self.precision, _dtheta(flat, self.theta, self.precision))
        if self.clip is None:
            self.clip = float(np.float32(2 * np.abs(self.a_ref).max() + 1.0))
        self.set_target(self.a_ref)

    def set_target(self, a):
        self.target = np.ascontiguousarray(a, dtype=np.float32)
        self.rounding = np.abs(np.clip(self.a_ref, -self.clip, self.clip) - self.target.astype(np.float64))
        self.t = torch.from_numpy(self.target).to(DEV)

    def first(self, plain=False):
        """The global index of this case's launch: its member, or mirrored the even member of its pair."""
        return 2 * self.member if self.mirrored and not plain else self.member

    def eval(self, target=None, n_local=None, member_offset=None, sigma=None, workspace=None, out=None, plain=False):
        """The case member's fitness [1] (mirrored: out[1] of its pair's launch, `out` then holds 2), or with n_local
        the fitness of members [member_offset, member_offset + n_local).  plain: des_nes_eval, mirrored case or not."""
        mirrored = self.mirrored and not plain
        one = n_local is None
        if one:
            n_local = 2 if mirrored else 1
        f = (ops().nes_eval_mirrored if mirrored else ops().nes_eval)(
            self.th, self.o, self.t if target is None else target, hidden=self.H,
            sigma=self.sigma if sigma is None else sigma, clip=self.clip, seed=SEED, generation=GEN,
            member_offset=self.first(plain) if member_offset is None else member_offset, n_local=n_local,
            precision=self.precision, workspace=workspace, out=out)
        return f[1:] if one and mirrored else f

    def tol(self):
        """Per-action tolerance on |e| (probes): KAPPA_PROBE * B plus the fp32 rounding of the target."""
        return KAPPA_PROBE[self.precision] * self.B + self.rounding

    def residual_limit(self):
        """-fitness may not exceed sum((KAPPA_RESIDUAL * B + target rounding)^2) (triangle inequality), plus the fp32
        rounding of the fitness."""
        return float(np.sum((KAPPA_RESIDUAL[self.precision] * self.B + self.rounding) ** 2)) * (1 + 2.0 ** -20)

    def depth(self):
        return fe.ffma_reduction_depth(self.A, self.T) if self.precision == 'fp32' else fe.tc_reduction_depth(self.A, self.T)

    def probe(self, entries):
        """Action errors e_r = a_gpu_r - target_r of the flat entries from one launch per entry."""
        d = fe.probe_offsets(self.target, entries)
        K = len(entries)
        tg = np.repeat(self.target[None], K, axis=0).reshape(K, -1)
        tg[np.arange(K), entries] = (tg[np.arange(K), entries].astype(np.float64) + d).astype(np.float32)
        tg_dev = torch.from_numpy(tg.reshape(K, self.T, self.A)).to(DEV)
        fits = torch.empty(K, 2 if self.mirrored else 1, dtype=torch.float32, device=DEV)
        for k in range(K):
            self.eval(target=tg_dev[k], out=fits[k])
        f0 = float(self.eval().item())
        f = fits[:, -1].cpu().numpy().astype(np.float64)
        return fe.probe_recover(f0, f, d), fe.probe_resolution(d, f0, f, self.depth()), f0


def _and_mirrored(params):
    """Each (values, id) plain under its own id, then mirrored under id + '-mirrored'; `mirrored` is the last argument."""
    return ([pytest.param(*v, False, id=i) for v, i in params] +
            [pytest.param(*v, True, id=i + '-mirrored') for v, i in params])


def _cases(precisions):
    return _and_mirrored([(c + (p,), 'd0=%d-H=%d-A=%d-T=%d-%s' % (c + (p,))) for c in fe.FORWARD_CASES for p in precisions])


# ---------------------------------------------------------------------------------------------------------------------
# 1. residual tapes over every instantiation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d0,H,A,T,precision,mirrored', _cases(fe.PRECISIONS))
def test_residual_tape_within_bound(d0, H, A, T, precision, mirrored):
    """Mirrored, the pair's launch is compared whole: with and without the workspace bit for bit, and its even member
    with plain member p bit for bit (the only check on the even member of the A > 4 and ragged-d0 kernels)."""
    c = Case(d0, H, A, T, precision, member=5 + d0, mirrored=mirrored)
    assert np.all(np.abs(c.a_ref) < c.clip / 2)                       # nothing clips
    f = c.eval(n_local=2 if mirrored else 1)
    f0 = float(f[-1].item())
    assert np.isfinite(f0) and f0 <= 0
    assert -f0 <= c.residual_limit(), (np.sqrt(-f0 / np.sum(c.B ** 2)), KAPPA_RESIDUAL[precision])
    if mirrored:
        assert torch.equal(f[:1], c.eval(plain=True))                 # even member 2p = plain member p
    if precision != 'fp32' and fe.tc_passes(T) > 1:
        ws = ops().eval_workspace(d0, H, A, T, precision, DEV)
        assert ws is not None
        assert torch.equal(f, c.eval(n_local=f.numel(), workspace=ws))   # cached weight tiles: bit-identical


# ---------------------------------------------------------------------------------------------------------------------
# persistent loop and cluster slots
# ---------------------------------------------------------------------------------------------------------------------
LOOP_SHAPES = [(24, 256, 4, 256), (17, 128, 7, 384)]                 # CL2 one pass; CL1 three passes, NA = 8


@pytest.mark.parametrize('n_local,mirrored', _and_mirrored([((n,), str(n)) for n in (67, 133, 300)]))
@pytest.mark.parametrize('precision', ['f16', 'f16x3'])
@pytest.mark.parametrize('d0,H,A,T', LOOP_SHAPES)
def test_sigma_zero_members_identical_across_persistent_loop(d0, H, A, T, precision, n_local, mirrored):
    """sigma = 0: every member evaluates theta.  n_local 67 leaves a partial grid of clusters, 133 and 300 send CTAs
    round the persistent loop two and three times: all fitnesses bit-identical and within the bound.  Mirrored, the
    launch holds whole pairs (68, 134, 300 from member 12), and both members of every pair give the plain bits."""
    c = Case(d0, H, A, T, precision, member=0, sigma=0.0, mirrored=mirrored)
    assert np.array_equal(c.flat, c.theta)
    ws = ops().eval_workspace(d0, H, A, T, precision, DEV)
    if mirrored:
        f = c.eval(n_local=n_local + n_local % 2, member_offset=12, workspace=ws).cpu().numpy()
        assert np.all(f == float(c.eval(plain=True).item())), np.unique(f)
    else:
        f = c.eval(n_local=n_local, member_offset=11, workspace=ws).cpu().numpy()
    assert np.all(f == f[0]), np.unique(f)
    assert -float(f[0]) <= c.residual_limit()


@pytest.mark.parametrize('precision,mirrored', _and_mirrored([((p,), p) for p in ('f16', 'f16x3')]))
@pytest.mark.parametrize('d0,H,A,T', LOOP_SHAPES)
def test_member_on_later_loop_trip_within_bound(d0, H, A, T, precision, mirrored):
    """sigma > 0, n_local = 300: members 133 and 299 are evaluated on a CTA's second or third trip through the loop
    (132 CTAs, or 66 clusters).  Their residual tapes hold, and they match a launch of that member alone.  Mirrored,
    from the even member 40, both are odd members, and match a launch of their pair alone."""
    base = 40
    for m in (133, 299):
        c = Case(d0, H, A, T, precision, member=(base + m) // 2 if mirrored else base + m, mirrored=mirrored)
        f = c.eval(n_local=300, member_offset=base).cpu().numpy()
        assert -float(f[m]) <= c.residual_limit()
        assert f[m] == float(c.eval().item())


TOP_CASES = [(24, 256, 4, 256, 'f16x3'), (3, 128, 7, 384, 'f16'), (17, 64, 5, 256, 'fp32')]   # CL2, CL1, FFMA


@pytest.mark.parametrize('d0,H,A,T,precision,mirrored',
                         _and_mirrored([(c, 'd0=%d-H=%d-A=%d-T=%d-%s' % c) for c in TOP_CASES]))
def test_top_of_member_range_within_bound(d0, H, A, T, precision, mirrored):
    """The last member a shard can hold: plain member 2^32 - 1; mirrored the pair at member_offset 2^32 - 2, whose odd
    member 2^32 - 1 has counter word 2^31 - 1.  The producers form member_offset + m in 64 bits before noise_word's
    shift: theta' must be the oracle's at that counter word, and the residual tape must hold."""
    p = 2 ** 31 - 1 if mirrored else 2 ** 32 - 1
    c = Case(d0, H, A, T, precision, member=p, mirrored=mirrored)
    eps = orc.noise(SEED, GEN, p, 1, orc.param_count(d0, H, A))[0]
    ref = orc.perturb(c.theta, -SIGMA if mirrored else SIGMA, eps)
    r = np.sqrt((np.pad(eps, (0, eps.size % 2)) ** 2).reshape(-1, 2).sum(-1)).repeat(2)[:eps.size]
    tol = SIGMA * (4e-6 * (1 + np.abs(eps)) + 2.0 ** -22 * np.log(2) / np.maximum(r, 1e-4)) + 1e-7   # test_gpu_ops' bound
    assert np.all(np.abs(c.flat.astype(np.float64) - ref) <= tol)
    f = float(c.eval().item())
    assert -f <= c.residual_limit(), np.sqrt(-f / np.sum(c.B ** 2))


# ---------------------------------------------------------------------------------------------------------------------
# 2. per-action probes, one case per instantiation (the single-pass shapes)
# ---------------------------------------------------------------------------------------------------------------------
PROBE_CASES = [c for c in fe.FORWARD_CASES if fe.tc_passes(c[3]) == 1]


def _probe_params():
    out = [(c + (p,), 'd0=%d-H=%d-A=%d-T=%d-%s' % (c + (p,))) for c in PROBE_CASES for p in ('f16', 'f16x3')]
    out += [(c + ('fp32',), 'd0=%d-H=%d-A=%d-T=%d-fp32' % c) for c in PROBE_CASES if c[1] != 256]
    return _and_mirrored(out)


@pytest.mark.parametrize('d0,H,A,T,precision,mirrored', _probe_params())
def test_probe_every_action_within_bound(d0, H, A, T, precision, mirrored):
    """|e_r| <= kappa B_r per action (max norm), e_r recovered from fitness values alone."""
    c = Case(d0, H, A, T, precision, member=3, mirrored=mirrored)
    entries = fe.probe_entries(T, A)
    e, res, _ = c.probe(entries)
    tol = c.tol().reshape(-1)[entries] + res
    assert np.all(np.abs(e) <= tol), (np.max(np.abs(e) / tol), int(entries[np.argmax(np.abs(e) / tol)]))


def test_mirrored_cases_run_every_instantiation():
    """The mirrored residual and probe cases between them launch all 24 eval_tc_mirrored_kernel<H, X3, CL, NA>, and the
    FFMA kernel's mirrored path at ragged d0 and at A other than 4."""
    mirrored = [p.values for p in _cases(fe.PRECISIONS) + _probe_params() if p.values[-1]]
    got = {fe.tc_instantiation(H, A, T, prec) for d0, H, A, T, prec, _ in mirrored if prec != 'fp32'}
    assert got == {(H, x3, cl, na) for H in (64, 128, 256) for x3 in (False, True) for cl in (1, 2) for na in (4, 8)}
    ffma = [(d0, A) for d0, H, A, T, prec, _ in mirrored if prec == 'fp32']
    assert any(d0 % 4 for d0, _ in ffma) and any(A != 4 for _, A in ffma)


@pytest.mark.parametrize('precision,mirrored', _and_mirrored([((p,), p) for p in fe.PRECISIONS]))
def test_checks_trip_on_one_wrong_action(precision, mirrored):
    """Sensitivity, on the device: move one target entry r by 2 kappa B_r and the probe must flag r; move it by
    2 kappa ||B||_2 and the residual assert must fail.  This is the smallest single wrong action each check is
    guaranteed to catch (headline shape, see the module docstring for the numbers in action units)."""
    d0, H, A, T = HEADLINE
    c = Case(d0, H, A, T, precision, member=3, mirrored=mirrored)
    rng = np.random.RandomState(0)
    r = int(rng.randint(0, T * A))
    tol, limit, target = c.tol().reshape(-1), c.residual_limit(), c.target.copy().reshape(-1)
    e, res, f0 = c.probe(np.array([r]))
    assert abs(e[0]) <= tol[r] + res[0]
    moved = target.copy()
    moved[r] = np.float32(moved[r] + 2 * (tol[r] + res[0]) + 4 * 2.0 ** -24 * abs(moved[r]))
    c.set_target(moved.reshape(T, A))
    e2, res2, _ = c.probe(np.array([r]))
    assert abs(e2[0]) > tol[r] + res2[0]                               # the probe flags it
    moved = target.copy()
    moved[r] = np.float32(moved[r] + 2 * np.sqrt(limit))
    f = float(c.eval(target=torch.from_numpy(moved.reshape(T, A)).to(DEV)).item())
    assert -f > limit                                                  # the residual assert fails


# ---------------------------------------------------------------------------------------------------------------------
# 3. the odd member's sign, at each place the producers apply it
# ---------------------------------------------------------------------------------------------------------------------
EDGE_SHAPES = [(24, 64, 4, 256), (3, 128, 7, 384)]                   # CL2 NA4; CL1 three passes NA8, generic W1


@pytest.mark.parametrize('precision', fe.PRECISIONS)
@pytest.mark.parametrize('d0,H,A,T', EDGE_SHAPES)
@pytest.mark.parametrize('group', GROUPS)
def test_residual_trips_on_one_group_without_the_sign(group, d0, H, A, T, precision):
    """Sensitivity, on the device: the tensor-core producers give the odd member its sign at six places (b1, b2 and
    W3' among the small arrays, b3, W1' by quads when d0 % 4 == 0 and by scalars otherwise, the W2' chunks).
    Reference the odd member as if one group had kept the even member's +sigma*eps: the residual assert on the real
    odd member must fail, so a sign dropped at any one place is seen.  The FFMA kernel applies the sign once, to
    sigma, and runs the same cases."""
    c = Case(d0, H, A, T, precision, member=3, mirrored=True)
    even = ops().nes_perturb_mirrored(c.th, 2, SIGMA, SEED, GEN, member_offset=2 * c.member).cpu().numpy()[0]
    wrong, g = c.flat.copy(), _group_slices(d0, H, A)[group]
    wrong[g] = even[g]
    c.set_flat(wrong)
    f = float(c.eval().item())
    assert -f > c.residual_limit(), np.sqrt(-f / c.residual_limit())


# ---------------------------------------------------------------------------------------------------------------------
# 4. clip and non-finite values
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision,mirrored', _and_mirrored([((p,), p) for p in fe.PRECISIONS]))
@pytest.mark.parametrize('d0,H,A,T', EDGE_SHAPES)
def test_clip_zero_scores_the_target_alone(d0, H, A, T, precision, mirrored):
    """clip = 0: every action clips to 0, the fitness is -sum t^2 up to fp32 summation (target indexing and the
    reduction, independent of the network).  Mirrored: two whole pairs."""
    c = Case(d0, H, A, T, precision, member=1, clip=0.0, mirrored=mirrored)
    f = c.eval(n_local=4 if mirrored else 3).cpu().numpy().astype(np.float64)
    s = float(np.sum(c.target.astype(np.float64) ** 2))
    assert np.all(np.abs(f + s) <= (c.depth() + 3) * 2.0 ** -24 * s), (f, -s)


@pytest.mark.parametrize('precision,mirrored', _and_mirrored([((p,), p) for p in fe.PRECISIONS]))
@pytest.mark.parametrize('d0,H,A,T', EDGE_SHAPES)
def test_partial_clip_residual_within_bound(d0, H, A, T, precision, mirrored):
    """clip = median |a_ref| and target = clip(a_ref): clip is 1-Lipschitz, so the residual bound still holds.  Fails
    if the clip is applied before + b3, asymmetrically or after the subtraction."""
    c = Case(d0, H, A, T, precision, member=2, mirrored=mirrored)
    c.clip = float(np.float32(np.median(np.abs(c.a_ref))))
    c.set_target(np.clip(c.a_ref, -c.clip, c.clip))
    clipped = np.mean(np.abs(c.a_ref) > c.clip)
    assert 0.4 < clipped < 0.6
    assert np.any(c.a_ref > c.clip) and np.any(c.a_ref < -c.clip)
    f = float(c.eval().item())
    assert -f <= c.residual_limit()


@pytest.mark.parametrize('where,mirrored', _and_mirrored([((w,), w) for w in ('b3', 'obs')]))
@pytest.mark.parametrize('precision', fe.PRECISIONS)
@pytest.mark.parametrize('d0,H,A,T', EDGE_SHAPES)
def test_nan_action_gives_nan_fitness(d0, H, A, T, precision, where, mirrored):
    """np.clip keeps NaN (config.py:29,37, utils.py:134), so a NaN in b3[q] or in one observation row must make the
    fitness NaN, as orc.tape_fitness gives; a clamp written fminf(fmaxf(v, -clip), clip) would score it -clip.
    Mirrored: both members of both pairs."""
    obs, target = orc.synthetic_tape(T, d0, A)
    theta = orc.synthetic_theta(d0, H, A)
    if where == 'b3':
        theta[orc.param_count(d0, H, A) - A + A // 2] = np.nan
    else:
        obs[T // 2 + 1, d0 - 1] = np.nan
    ref = (mo if mirrored else orc).evaluate_population(theta, obs, target, SIGMA, 1.0, SEED, GEN, 0, 2, d0, H, A)
    assert np.all(np.isnan(ref))
    got = (ops().nes_eval_mirrored if mirrored else ops().nes_eval)(
        torch.from_numpy(theta).to(DEV), torch.from_numpy(obs).to(DEV), torch.from_numpy(target).to(DEV), hidden=H,
        sigma=SIGMA, clip=1.0, seed=SEED, generation=GEN, n_local=4 if mirrored else 3, precision=precision).cpu().numpy()
    assert np.all(np.isnan(got)), got
    if precision == 'fp32' and not mirrored:       # explicit weight vectors (CMA-ES) share the FFMA epilogue
        sol = torch.from_numpy(np.repeat(theta[None], 2, axis=0)).to(DEV)
        got = ops().pop_eval(sol, torch.from_numpy(obs).to(DEV), torch.from_numpy(target).to(DEV), hidden=H, clip=1.0)
        assert bool(torch.isnan(got).all())
