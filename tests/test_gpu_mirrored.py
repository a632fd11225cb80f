"""Mirrored (antithetic) sampling on the device: members 2p and 2p+1 are theta +- sigma*eps_p (include/des_b200.h).

* Tape forward: member 2p is bit-equal to plain member p on every kernel shape (fp32; f16 / f16x3 on 2-CTA clusters,
  single-CTA and multi-pass tapes, with and without the tile workspace); member 2p+1 matches the fp32 forward of the
  des_nes_perturb_mirrored rows within the per-precision tolerances of test_gpu_ops.py.  Every action of member 2p+1,
  on every eval kernel instantiation and against fp64, is checked in tests/test_gpu_forward_error.py.
* Rows, the pair-form reduction (against an fp64 sum over the device's own normals), closed-loop and host-stepped
  Pendulum and graph capture.  natural_es.train against the reference's verbatim run on explicit +-eps pairs is in
  tests/test_gpu_goldens.py, two GPUs in tests/test_gpu_multi.py."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import mirrored_oracle as mo
from oracle import nes_oracle as orc
from oracle import pendulum_oracle as po

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = {'fp32': 2e-5, 'f16x3': 3e-5, 'f16': 4e-3}
RTOL = 2e-4


def ops():
    from distributedes_b200 import ops as o
    return o


def dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).to(DEV)


# T = 256: 2-CTA cluster, one pass; 128: single CTA; 384: single CTA, three passes; 512: 2-CTA cluster, two passes
@pytest.mark.parametrize('T', [128, 256, 384, 512])
@pytest.mark.parametrize('H', [64, 128, 256])
@pytest.mark.parametrize('precision', ['fp32', 'f16', 'f16x3'])
def test_tape_forward_pairs(precision, H, T):
    d0, A, pairs, off = 24, 4, 40, 6
    obs, target = orc.synthetic_tape(T, d0, A)
    th, o, t = dev(orc.synthetic_theta(d0, H, A)), dev(obs), dev(target)
    kw = dict(hidden=H, sigma=0.1, clip=1.0, seed=9, generation=2, precision=precision)
    plain = ops().nes_eval(th, o, t, member_offset=off // 2, n_local=pairs, **kw)
    ws = ops().eval_workspace(d0, H, A, T, precision, DEV) if precision != 'fp32' else None
    for workspace in ([None, ws] if ws is not None else [None]):
        mir = ops().nes_eval_mirrored(th, o, t, member_offset=off, n_local=2 * pairs, workspace=workspace, **kw)
        assert torch.equal(mir[0::2], plain), workspace is not None
    rows = ops().nes_perturb_mirrored(th, 2 * pairs, 0.1, 9, 2, member_offset=off)
    ref = ops().pop_eval(rows[1::2].contiguous(), o, t, hidden=H, clip=1.0)
    rel = ((mir[1::2] - ref).abs() / ref.abs()).max().item()
    assert rel < TOL[precision], rel


def test_perturb_rows():
    P, pairs, off = 6020, 12, 10
    theta = dev(orc.synthetic_theta(24, 64, 4))
    rows = ops().nes_perturb_mirrored(theta, 2 * pairs, 0.1, 3, 5, member_offset=off)
    plain = ops().nes_perturb(theta, pairs, 0.1, 3, 5, member_offset=off // 2)
    assert torch.equal(rows[0::2], plain)
    eps = ops().noise_fill(pairs, P, 3, 5, member_offset=off // 2).double()
    ref = (theta.double() - float(np.float32(0.1)) * eps).float()
    ulp = (torch.nextafter(ref, torch.full_like(ref, np.inf)) - ref).abs()
    assert bool(((rows[1::2] - ref).abs() <= ulp).all())


def _pair_reference(shaped, P, seed, gen, member_offset, chunk=2048):
    s = shaped.double()
    c = s[0::2] - s[1::2]
    g = torch.zeros(P, dtype=torch.float64, device=DEV)
    for o in range(0, c.numel(), chunk):
        n = min(chunk, c.numel() - o)
        g += c[o:o + n] @ ops().noise_fill(n, P, seed, gen, member_offset=member_offset // 2 + o).double()
    return g


@pytest.mark.parametrize('P', [6020, 73220])
@pytest.mark.parametrize('N', [64, 4096, 65536])
def test_pair_form_reduction(N, P):
    rs = np.random.RandomState(N + P)
    shaped = dev(orc.fitness_shift(rs.randn(N)))
    kw = dict(seed=12, generation=3)
    got = ops().nes_grad_partial_mirrored(shaped, P, **kw).double()
    ref = _pair_reference(shaped, P, 12, 3, 0)
    assert ((got - ref).norm() / ref.norm()).item() <= 1e-5
    assert ((got - ref).abs().max() / ref.abs().max()).item() <= 1e-5
    # shards at even offsets sum to the whole
    cuts = [0, 2 * (N // 6), 2 * (N // 3), N]
    parts = sum(ops().nes_grad_partial_mirrored(shaped[a:b].contiguous(), P, member_offset=a, **kw).double()
                for a, b in zip(cuts[:-1], cuts[1:]))
    assert ((parts - ref).norm() / ref.norm()).item() <= 1e-5
    # the plain workspace query sizes the mirrored call; a short workspace is DES_ERR_WORKSPACE
    ws = ops().grad_workspace(N, P, DEV)
    assert torch.equal(ops().nes_grad_partial_mirrored(shaped, P, workspace=ws, **kw).double(), got)
    with pytest.raises(RuntimeError, match='status -4'):
        ops().nes_grad_partial_mirrored(shaped, P, workspace=torch.empty(16, dtype=torch.uint8, device=DEV), **kw)


@pytest.mark.parametrize('H', [16, 32, 64, 96, 128])
def test_closed_loop_equals_explicit_rows(H):
    n, off, reps, seed, gen = 12, 4, 10, 21, 3
    theta = dev(orc.synthetic_theta(3, H, 1, seed=H))
    st = dev(np.array([-0.2, 0.01, 0.3, 0.5, 0.4, 20.0, 32000.0], np.float32))
    kw = dict(hidden=H, horizon=120, repetitions=reps, clip=2.0, action_noise_std=0.2, seed=seed, generation=gen,
              member_offset=off, obs_stats=st)
    tot_a = torch.zeros(7, dtype=torch.float64, device=DEV)
    tot_b = torch.zeros(7, dtype=torch.float64, device=DEV)
    a = ops().rollout_eval_mirrored(theta, sigma=0.1, n_local=n, totals_out=tot_a, **kw)
    rows = ops().nes_perturb_mirrored(theta, n, 0.1, seed, gen, member_offset=off)
    b = ops().rollout_eval_solutions(rows, totals_out=tot_b, **kw)
    assert torch.equal(a, b) and torch.equal(tot_a, tot_b)
    # shard invariance: [off, off + 4) + [off + 4, off + n) in two launches
    kw.pop('member_offset')
    lo = ops().rollout_eval_mirrored(theta, sigma=0.1, n_local=4, member_offset=off, **kw)
    hi = ops().rollout_eval_mirrored(theta, sigma=0.1, n_local=n - 4, member_offset=off + 4, **kw)
    assert torch.equal(a, torch.cat([lo, hi]))
    with pytest.raises(RuntimeError, match='whole pairs'):
        ops().rollout_eval_mirrored(theta, sigma=0.1, n_local=3, member_offset=off, **kw)


def test_host_stepped_pendulum_equals_closed_loop():
    """HostEnvEngine(mirrored=True) stepping Pendulum-v0 on the host evaluates the members RolloutEngine(mirrored=True)
    evaluates on the device, and both match the oracle's mirrored closed-loop fitness."""
    from distributedes_b200.engine import HostEnvEngine, RolloutEngine
    H, N, reps, seed = 32, 12, 3, 5
    theta0 = orc.synthetic_theta(3, H, 1, seed=4)
    kw = dict(hidden=H, pop_size=N, theta0=theta0, sigma=0.1, learning_rate=0.1, repetitions=reps, seed=seed,
              mirrored=True)
    host = HostEnvEngine(env_fn=None, state_dim=3, action_dim=1, batch_env_fn=lambda B: po.PendulumBatch(B, seed),
                         clip=2.0, **kw)
    roll = RolloutEngine(**kw)
    fh, fr = host.evaluate().cpu().numpy(), roll.evaluate().cpu().numpy()
    assert host.steps_taken == N * reps * po.HORIZON
    assert np.max(np.abs(fh - fr) / np.abs(fr)) < RTOL
    ref, _ = mo.closed_fitness(theta0, H, 0.1, seed, 0, 0, N, reps)
    assert np.max(np.abs(fh - ref) / np.abs(ref)) < RTOL
    assert np.array_equal(host.rows[0::2].cpu().numpy(), ops().nes_perturb(dev(theta0), N // 2, 0.1, seed, 0).cpu().numpy())


@pytest.mark.parametrize('precision', ['f16x3', 'f16'])
def test_graph_captured_generation_equals_eager(precision):
    from distributedes_b200.engine import NESEngine
    d0, H, A, T, N = 24, 64, 4, 256, 400
    obs, target = orc.synthetic_tape(T, d0, A)
    kw = dict(state_dim=d0, hidden=H, action_dim=A, pop_size=N, theta0=orc.synthetic_theta(d0, H, A), obs=obs,
              target=target, sigma=0.1, learning_rate=0.05, seed=3, precision=precision, device=DEV, mirrored=True)
    a, b = NESEngine(use_graph=True, **kw), NESEngine(use_graph=False, **kw)
    for _ in range(3):
        a.generation()
        b.generation()
        assert torch.equal(a.fitness_all, b.fitness_all) and torch.equal(a.theta, b.theta)
    assert not torch.equal(a.theta, torch.from_numpy(kw['theta0']).to(DEV))
