"""rollout_pendulum_kernel action by action: every step of every episode recovered from the public outputs and checked
against the fp64 forward of the member's own weights.

The return checks of test_gpu_rollout.py / test_gpu_cma_rollout.py (|dR|/|R| < 2e-4) see the policy only through 200
steps of a feedback loop.  Here the loop is opened (oracle/rollout_probe.py): launches with horizons h and repetitions
r = 1..10 give fp64 observation totals whose double differences are the kernel's fp32 observations at every step of
every episode, and gym's dynamics then give the torque u_rec the environment applied at each step, to ~3e-6
(``resolution``).  Each one must satisfy

    |u_rec - clamp_2(clip(a*))| <= KAPPA * B + resolution,

a* the fp64 forward (plus the oracle's action noise) of the member's weights at the kernel's own normalised observation,
B = oracle.forward_error.closed_loop_bound ('mufu': fp32 FFMA chains, tanh_mufu, the fp32 normaliser, the layer-3
butterfly).  B is a worst-case bound that grows with the width (H FFMA roundings per unit, H units into the action)
while the kernel's real error stays below the recovery resolution at every width: the largest |u_rec - clamp_2(clip(a*))|
of every case is 2.4e-6 to 3.4e-6, all of it resolution.  KAPPA is therefore set per width from the measured maximum of
|u_rec - clamp_2(clip(a*))| / B over the cases of this file at that width (one run on an H100 80GB HBM3, 700 W power
limit), rounded up from 4x:

    H      cases (max |d| / B)                                                        max      KAPPA
    16     nes-h16 0.404, rows-h16 0.311                                              0.404    1.7
    32     nes-h32 0.104, nes-h32-noise 0.092, mirrored-h32 0.118, clip-3.0 0.056     0.118    0.5
    64     nes-h64 0.035, nes-h64-stats 0.028, clip-0.5 0.030, top-member 0.032       0.035    0.15
    96     nes-h96 0.011, rows-h96-stats-noise 0.0037                                 0.011    0.045
    128    nes-h128 0.0068, nes-h128-stats-noise 0.0065, mirrored-h128-stats-noise 0.0069   0.0069   0.028

The kernels are deterministic, so the maxima repeat run to run; the 4x covers other compilers and drivers.  So an action
off by 3e-6 + KAPPA B fails: 1.6e-5 to 1.7e-5 at the median B of every width.

Sensitivity (test_checks_trip_on_a_wrong_policy, nes-h64, all 200 steps of all 10 episodes), same run:

    oracle                                   max |d| / (KAPPA B + res)    return |dR|/|R| (the 2e-4 check)
    exact                                    0.19                         4.3e-8   passes
    one W2 entry moved by 2^-10              7.1                          2.5e-5   passes: misses it
    tanh with tanh.approx's 2^-11 rel. error 62                           2.0e-3   trips

The W2 change moves actions by up to ~1e-4 and the returns by 2.5e-5, eight times under the return check's bar; the
per-action check flags it with a margin of 7.
"""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import forward_error as fe
from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po
from oracle import rollout_probe as rp

pytestmark = pytest.mark.gpu

SEED, GEN, SIGMA = 2026, 4, 0.1
KAPPA = {16: 1.7, 32: 0.5, 64: 0.15, 96: 0.045, 128: 0.028}          # per hidden width, see above
RETURN_RTOL = 2e-4                  # test_gpu_rollout.py's return check
STATS = (np.float32([-0.2, 0.01, 0.3]), np.float32([0.5, 0.4, 20.0]), np.float32(32000))
ALL = range(0, 200)
WIDE = list(range(0, 41)) + list(range(180, 200))
SHORT = range(0, 41)
TOP = (1 << 28) - 1                 # the last member the action-noise counter member*16 + episode can address

# id: (mode, H, steps, stats, action noise, clip, member)
CASES = {
    'nes-h16': ('nes', 16, ALL, None, 0.0, 2.0, 3),
    'nes-h32': ('nes', 32, ALL, None, 0.0, 2.0, 3),
    'nes-h64': ('nes', 64, ALL, None, 0.0, 2.0, 3),
    'nes-h96': ('nes', 96, ALL, None, 0.0, 2.0, 3),
    'nes-h128': ('nes', 128, ALL, None, 0.0, 2.0, 3),
    'nes-h64-stats': ('nes', 64, WIDE, STATS, 0.0, 2.0, 11),
    'nes-h32-noise': ('nes', 32, ALL, None, 0.3, 2.0, 6),
    'nes-h128-stats-noise': ('nes', 128, WIDE, STATS, 0.3, 2.0, 6),
    'rows-h16': ('rows', 16, ALL, None, 0.0, 2.0, 40),
    'rows-h96-stats-noise': ('rows', 96, WIDE, STATS, 0.3, 2.0, 41),
    'mirrored-h32': ('mirrored', 32, WIDE, None, 0.0, 2.0, 7),
    'mirrored-h128-stats-noise': ('mirrored', 128, WIDE, STATS, 0.3, 2.0, 9),
    'clip-0.5': ('nes', 64, SHORT, None, 0.0, 0.5, 5),
    'clip-3.0': ('rows', 32, SHORT, None, 0.3, 3.0, 5),
    'top-member': ('nes', 64, SHORT, None, 0.3, 2.0, TOP),
}


def ops():
    from distributedes_b200 import ops as _ops
    return _ops


def dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).cuda()


def _stats_tensor(stats):
    return None if stats is None else dev(np.concatenate([stats[0], stats[1], [stats[2]]]))


def _theta(H):
    return orc.synthetic_theta(3, H, 1, seed=H)


def _solution(H, member):
    """An explicit solution row, as CMA-ES's ask() would return: theta plus a wide Gaussian step."""
    rs = np.random.RandomState(member)
    return (_theta(H) + 0.3 * rs.randn(orc.param_count(3, H, 1))).astype(np.float32)


class Probe:
    """One member's 10 episodes recovered from the totals of launches (horizon h, repetitions r), one member each."""

    def __init__(self, mode, H, steps, stats, noise, clip, member):
        o = ops()
        self.mode, self.H, self.stats, self.noise, self.clip, self.member = mode, H, stats, noise, clip, member
        self.steps = np.asarray(sorted(steps))
        self.hs = rp.horizons(self.steps)
        st = _stats_tensor(stats)
        P = orc.param_count(3, H, 1)
        theta = dev(_theta(H))
        kw = dict(hidden=H, clip=clip, action_noise_std=noise, seed=SEED, generation=GEN, obs_stats=st)
        ws = torch.empty(2 * 7, dtype=torch.float64, device='cuda')
        fit = torch.empty(2, dtype=torch.float32, device='cuda')

        def table(launch):
            T = torch.zeros((len(self.hs), rp.EPISODES, 7), dtype=torch.float64, device='cuda')
            for i, h in enumerate(self.hs):
                for r in range(1, rp.EPISODES + 1):
                    launch(h, r, T[i, r - 1])
            return T.cpu().numpy()

        if mode == 'nes':
            self.row = o.nes_perturb(theta, 1, SIGMA, SEED, GEN, member_offset=member)
            T = table(lambda h, r, out: o.rollout_eval(theta, horizon=h, repetitions=r, sigma=SIGMA, member_offset=member,
                                                       n_local=1, totals_out=out, workspace=ws, out=fit[:1], **kw))
            mag = None
        elif mode == 'rows':
            self.row = dev(_solution(H, member)).reshape(1, P)
            T = table(lambda h, r, out: o.rollout_eval_solutions(self.row, horizon=h, repetitions=r, member_offset=member,
                                                                 totals_out=out, workspace=ws, out=fit[:1], **kw))
            mag = None
        else:
            # an odd member (-sigma) of a mirrored pair: the pair's totals minus its even member's, which the rows
            # path evaluates to the same bits (DESIGN §4.7)
            assert member % 2 == 1
            pair = o.nes_perturb_mirrored(theta, 2, SIGMA, SEED, GEN, member_offset=member - 1)
            self.row = pair[1:].contiguous()
            Tp = table(lambda h, r, out: o.rollout_eval_mirrored(theta, horizon=h, repetitions=r, sigma=SIGMA,
                                                                 member_offset=member - 1, n_local=2, totals_out=out,
                                                                 workspace=ws, out=fit, **kw))
            even = pair[:1].contiguous()
            Te = table(lambda h, r, out: o.rollout_eval_solutions(even, horizon=h, repetitions=r, member_offset=member - 1,
                                                                  totals_out=out, workspace=ws, out=fit[:1], **kw))
            T, mag = Tp - Te, np.abs(Tp) + np.abs(Te)
        self.totals = T
        self.flat = self.row.cpu().numpy().reshape(-1)
        self.obs, self.err = rp.observations(T, self.hs, mag=mag)
        self.u_all, self.res_all, valid = rp.torques(self.obs, self.err)
        t = self.steps
        self.u, self.res, self.valid = self.u_all[:, t], self.res_all[:, t], valid[:, t]
        self.std32 = float(np.float32(noise))
        z0, z1 = rp.action_normals(SEED, GEN, member, int(t.max()) + 1)
        self.nz = self.std32 * z0[:, t]
        self.nerr = self.std32 * rp.normal_error(z0[:, t], z1[:, t])

    def actions(self, flat=None, tanh=np.tanh):
        """a* [10, steps] at the kernel's own observations."""
        x = self.obs[:, self.steps]
        return fe.closed_loop_actions(self.flat if flat is None else flat, x, 3, self.H, 1, self.stats,
                                      self.nz[..., None], tanh=tanh)[..., 0]

    def bound(self):
        x = self.obs[:, self.steps]
        return fe.closed_loop_bound(self.flat, x, 3, self.H, 1, self.stats, self.nz[..., None],
                                    self.nerr[..., None])[..., 0]

    def deviation(self, a):
        """|u_rec - clamp_2(clip(a))| at the valid steps (others 0)."""
        return np.where(self.valid, np.abs(self.u - rp.applied(a, self.clip)), 0.0)

    def returns(self, horizon=200):
        """The device's episode returns [10] of this member (one launch, all repetitions)."""
        o = ops()
        ep = torch.empty(rp.EPISODES * (2 if self.mode == 'mirrored' else 1), dtype=torch.float32, device='cuda')
        kw = dict(hidden=self.H, horizon=horizon, repetitions=rp.EPISODES, clip=self.clip, action_noise_std=self.noise,
                  seed=SEED, generation=GEN, obs_stats=_stats_tensor(self.stats), episodes_out=ep)
        if self.mode == 'nes':
            o.rollout_eval(dev(_theta(self.H)), sigma=SIGMA, member_offset=self.member, n_local=1, **kw)
        elif self.mode == 'rows':
            o.rollout_eval_solutions(self.row, member_offset=self.member, **kw)
        else:
            o.rollout_eval_mirrored(dev(_theta(self.H)), sigma=SIGMA, member_offset=self.member - 1, n_local=2, **kw)
        return ep.cpu().numpy().astype(np.float64)[-rp.EPISODES:]


_PROBES = {}


def probe(name):
    if name not in _PROBES:
        _PROBES[name] = Probe(*CASES[name])
    return _PROBES[name]


@pytest.mark.parametrize('name', list(CASES))
def test_episodes_reset_and_step_as_the_oracle_says(name):
    """Step 0 of every episode is fp32 of pendulum_oracle.reset_states (one ulp: device fp64 sincos against numpy's),
    the observation counts are r * h exactly, and from (th, thdot, u_rec) pendulum_step predicts the next observation
    within its rounding: the device environment, step by step, free of the feedback."""
    p = probe(name)
    ref = rp.reset_observations(SEED, GEN, p.member).astype(np.float64)
    got = p.obs[:, 0]
    assert np.all(np.abs(got - ref) <= np.spacing(np.abs(ref).astype(np.float32))), np.abs(got - ref).max()
    assert np.array_equal(p.totals[..., 6], np.outer(p.hs, np.arange(1, rp.EPISODES + 1)))
    t = p.steps
    pred = rp.predict(p.obs, p.u_all)[:, t]
    nxt = p.obs[:, t + 1]
    tol = rp.predict_tolerance(p.obs, p.res_all)[:, t]
    ok = p.valid[..., None] & np.isfinite(nxt)
    assert np.all((np.abs(pred - nxt) <= tol)[ok]), np.max(np.where(ok, np.abs(pred - nxt) / tol, 0))
    assert p.valid.mean() > 0.5


@pytest.mark.parametrize('name', list(CASES))
def test_every_action_within_the_bound(name):
    p = probe(name)
    a, B = p.actions(), p.bound()
    d = p.deviation(a)
    ratio = np.max(d / B)
    print('\nRATIO %s max|d|/B %.4g  max|d| %.3g  median B %.3g  median res %.3g  steps checked %d' %
          (name, ratio, d.max(), np.median(B), np.median(p.res), int(p.valid.sum())))
    assert np.all(d <= KAPPA[p.H] * B + p.res), np.max((d - p.res) / B)


@pytest.mark.parametrize('name', ['nes-h16', 'nes-h64-stats', 'nes-h128-stats-noise', 'rows-h96-stats-noise',
                                  'mirrored-h32', 'clip-0.5', 'clip-3.0', 'top-member'])
def test_policy_act_computes_the_rollout_action(name):
    """DESIGN §4.8: des_policy_act gives the rollout kernel's action for the same observation and weights.  Fed the
    recovered observations, the member's row and step index, its clipped actions match u_rec within the recovery
    resolution alone."""
    p = probe(name)
    o = ops()
    st = _stats_tensor(p.stats)
    alive = torch.ones((1, rp.EPISODES), dtype=torch.uint8, device='cuda')
    acts = torch.empty((len(p.steps), 1, rp.EPISODES, 1), dtype=torch.float32, device='cuda')
    obs = dev(p.obs[:, p.steps].transpose(1, 0, 2).astype(np.float32))
    for i, t in enumerate(p.steps):
        o.policy_act(p.row, obs[i].contiguous(), alive, state_dim=3, hidden=p.H, action_dim=1,
                     repetitions=rp.EPISODES, clip=p.clip, action_noise_std=p.noise, seed=SEED, generation=GEN,
                     member_offset=p.member, t=int(t), obs_stats=st, out=acts[i])
    act = acts.cpu().numpy()[:, 0, :, 0].T.astype(np.float64)
    d = np.where(p.valid, np.abs(p.u - np.clip(act, -2.0, 2.0)), 0.0)
    assert np.all(d <= p.res), np.max(d / p.res)


def test_checks_trip_on_a_wrong_policy():
    """Sensitivity: the per-action check fails against an oracle with one W2 entry moved by 2^-10 (the unit with the
    largest |W3|, its largest input weight) and against one whose tanh carries tanh.approx's 2^-11 relative error.
    Printed beside it: what the 2e-4 return check makes of the same oracles."""
    p = probe('nes-h64')
    B = p.bound()
    lim = KAPPA[p.H] * B + p.res
    H = p.H
    W1, b1, W2, b2, W3, b3 = orc.unflatten(p.flat.astype(np.float64), 3, H, 1)
    j = int(np.argmax(np.abs(W3[0])))
    k = int(np.argmax(np.abs(W2[j])))
    moved = p.flat.copy()
    moved[3 * H + H + j * H + k] += np.float32(2.0 ** -10)
    approx = lambda z: np.tanh(z) * (1 + 2.0 ** -11)
    dev_ret = p.returns()
    report = []
    for tag, flat, tanh in (('exact', None, np.tanh), ('w2', moved, np.tanh), ('tanh', None, approx)):
        d = p.deviation(p.actions(flat, tanh))
        ret, _, _, _ = po.rollouts((p.flat if flat is None else flat).reshape(1, -1), H, SEED, GEN, [p.member],
                                   rp.EPISODES, None, 200, p.clip, 0.0, tanh=tanh)
        rel = np.max(np.abs(dev_ret - ret[0]) / np.abs(ret[0]))
        report.append((tag, np.max(d / lim), rel))
        print('\nSENSITIVITY %s  max |d| / (kappa B + res) %.3g  return |dR|/|R| %.3g (trips at %g: %s)' %
              (tag, np.max(d / lim), rel, RETURN_RTOL, rel >= RETURN_RTOL))
    exact, w2, tn = report
    assert exact[1] <= 1 and exact[2] < RETURN_RTOL
    assert w2[1] > 1 and tn[1] > 1


def test_horizon_one_and_every_repetition_count():
    """horizon = 1 (one observation, one reward) at every repetition count, four members at once: fitness and
    episode returns equal the oracle's first-step rewards to fp32 rounding."""
    o = ops()
    H, n = 32, 4
    theta = _theta(H)
    for reps in range(1, rp.EPISODES + 1):
        ep = torch.empty(n * reps, dtype=torch.float32, device='cuda')
        fit = o.rollout_eval(dev(theta), hidden=H, horizon=1, repetitions=reps, sigma=SIGMA, clip=2.0, seed=SEED,
                             generation=GEN, member_offset=8, n_local=n, episodes_out=ep)
        ref, _ = po.closed_fitness(theta, H, SIGMA, SEED, GEN, 8, n, reps, None, 1)
        eps = orc.noise(SEED, GEN, 8, n, orc.param_count(3, H, 1))
        ret, _, _, _ = po.rollouts(orc.perturb(theta, SIGMA, eps), H, SEED, GEN, np.arange(8, 8 + n), reps, None, 1)
        assert np.allclose(fit.cpu().numpy(), ref, rtol=1e-6, atol=1e-6)
        assert np.allclose(ep.cpu().numpy().reshape(n, reps), ret, rtol=1e-6, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# NaN actions: np.clip keeps NaN (config.py:29, utils.py:134, gym's Pendulum), so a NaN action gives a NaN return
# ---------------------------------------------------------------------------------------------------------------------
def _poisoned(H, where):
    flat = _theta(H).copy()
    P = flat.size
    w3 = P - 1 - H
    if where == 'b3-nan':
        flat[P - 1] = np.nan
    elif where == 'w3-nan':
        flat[w3 + 2] = np.nan
    elif where == 'w3-inf-pair':                     # +inf and -inf on two units: inf - inf wherever their signs agree
        flat[w3 + 1], flat[w3 + 5] = np.inf, -np.inf
    return flat


@pytest.mark.parametrize('where', ['b3-nan', 'w3-nan', 'w3-inf-pair'])
@pytest.mark.parametrize('H', [16, 64])
def test_nan_action_gives_nan_fitness_on_the_closed_loop(H, where):
    """A member with a NaN b3, a NaN W3 entry or opposite infinities in W3 gets NaN episode returns and a NaN fitness
    from rollout_eval, rollout_eval_mirrored and rollout_eval_solutions, as the oracle does; its neighbours (explicit
    rows) keep their fitness bit for bit."""
    o = ops()
    n, reps, horizon, off = 4, 10, 60, 2
    bad = _poisoned(H, where)
    ref, _, _, _ = po.rollouts(bad.reshape(1, -1), H, SEED, GEN, [off + 1], reps, None, horizon)
    assert np.isnan(ref).all()
    kw = dict(hidden=H, horizon=horizon, repetitions=reps, clip=2.0, seed=SEED, generation=GEN)
    # NES: every member perturbs the poisoned theta (theta + sigma*eps keeps NaN and inf); with opposite infinities an
    # episode whose two units never agree in sign stays finite, in the oracle as on the device
    P = orc.param_count(3, H, 1)
    for fn, eps in ((o.rollout_eval, orc.noise(SEED, GEN, off, n, P)),
                    (o.rollout_eval_mirrored, mo.noise_mirrored(SEED, GEN, off, n, P))):
        ep = torch.empty(n * reps, dtype=torch.float32, device='cuda')
        fit = fn(dev(bad), sigma=SIGMA, member_offset=off, n_local=n, episodes_out=ep, **kw)
        ref_ep, _, _, _ = po.rollouts(orc.perturb(bad, SIGMA, eps), H, SEED, GEN, np.arange(off, off + n), reps, None,
                                      horizon)
        assert np.isnan(ref_ep.mean(1)).all() and torch.isnan(fit).all(), (fn.__name__, fit)
        assert np.array_equal(torch.isnan(ep).cpu().numpy().reshape(n, reps), np.isnan(ref_ep)), fn.__name__
    # explicit rows: only row 1 is poisoned
    rows = np.stack([_solution(H, 100 + i) for i in range(n)])
    clean = o.rollout_eval_solutions(dev(rows), member_offset=off, **kw).clone()
    rows[1] = bad
    ep = torch.empty(n * reps, dtype=torch.float32, device='cuda')
    fit = o.rollout_eval_solutions(dev(rows), member_offset=off, episodes_out=ep, **kw)
    assert torch.isnan(fit[1]) and torch.isnan(ep.reshape(n, reps)[1]).all()
    keep = [0, 2, 3]
    assert torch.equal(fit[keep], clean[keep]) and not torch.isnan(ep.reshape(n, reps)[keep]).any()


def test_one_infinite_w3_entry_clips_like_the_oracle():
    """np.clip(inf) is the clip: a single +inf W3 entry saturates the action, the return stays finite and matches."""
    o = ops()
    H, reps, horizon = 32, 4, 60
    flat = _theta(H).copy()
    flat[flat.size - 1 - H + 3] = np.inf
    ep = torch.empty(reps, dtype=torch.float32, device='cuda')
    o.rollout_eval_solutions(dev(flat.reshape(1, -1)), hidden=H, horizon=horizon, repetitions=reps, clip=2.0,
                             seed=SEED, generation=GEN, member_offset=0, episodes_out=ep)
    ref, _, _, _ = po.rollouts(flat.reshape(1, -1), H, SEED, GEN, [0], reps, None, horizon)
    got = ep.cpu().numpy()
    assert np.isfinite(ref).all() and np.isfinite(got).all()
    assert np.allclose(got, ref[0], rtol=RETURN_RTOL)


@pytest.mark.parametrize('H', [16, 96, 128])
def test_policy_act_keeps_nan(H):
    """policy_act: an alive slot with a NaN observation gets a NaN action, a member with NaN weights NaN actions in
    every alive slot; dead slots still get 0, and the other slots keep their actions bit for bit."""
    o = ops()
    n, reps = 3, 6
    rows = np.stack([_solution(H, 200 + i) for i in range(n)])
    rs = np.random.RandomState(H)
    obs = rs.uniform(-1, 1, (n, reps, 3)).astype(np.float32)
    alive = np.ones((n, reps), np.uint8)
    alive[0, 4] = 0
    kw = dict(state_dim=3, hidden=H, action_dim=1, repetitions=reps, clip=2.0, seed=SEED, generation=GEN, t=5)
    clean = o.policy_act(dev(rows), dev(obs), dev(alive, torch.uint8), **kw).cpu().numpy()
    obs[0, 2, 1] = np.nan                            # alive slot
    obs[0, 4, 0] = np.nan                            # dead slot
    rows[2, orc.param_count(3, H, 1) - 1] = np.nan   # member 2's b3
    got = o.policy_act(dev(rows), dev(obs), dev(alive, torch.uint8), **kw).cpu().numpy()
    assert np.isnan(got[0, 2]).all() and got[0, 4, 0] == 0.0 and np.isnan(got[2]).all()
    same = np.ones((n, reps), bool)
    same[0, 2] = same[2, :] = False
    assert np.array_equal(got[same], clean[same])
