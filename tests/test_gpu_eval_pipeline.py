"""The tensor-core evaluation is a persistent, warp-specialised pipeline: a producer warpgroup generates the next
member's weights while the consumer warpgroups still run the current one, through double-buffered shared memory.  A
member's fitness must not depend on which member its CTA evaluated before it, on which CTA it lands on, or on whether
the multi-pass W2' chunks come from the workspace mirror or are regenerated.  Every FORWARD_CASES shape (so every
eval_tc_kernel instantiation, one- and multi-pass) is checked bit for bit over several trips of the persistent loop."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import forward_error as fe
from oracle import nes_oracle as orc

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
SEED, GEN, SIGMA = 77, 5, 0.1
N_LOCAL = 300                                           # > 2 x 132 CTAs: three trips of the persistent loop
SHARDS = ((1, 7), (65, 140), (133, 167))                # other CTAs, other predecessors, partial last waves


def _params():
    return [pytest.param(*c, p, id='d0=%d-H=%d-A=%d-T=%d-%s' % (c + (p,))) for c in fe.FORWARD_CASES for p in ('f16', 'f16x3')]


@pytest.mark.parametrize('d0,H,A,T,precision', _params())
def test_fitness_independent_of_predecessor_and_cta(d0, H, A, T, precision):
    from distributedes_b200 import ops
    obs, target = orc.synthetic_tape(T, d0, A, seed=7 * T + d0)
    theta = torch.from_numpy(orc.synthetic_theta(d0, H, A, seed=H + A + 1)).to(DEV)
    o, t = torch.from_numpy(obs).to(DEV), torch.from_numpy(target).to(DEV)
    ws = ops.eval_workspace(d0, H, A, T, precision, DEV)

    def run(off, n, workspace):
        return ops.nes_eval(theta, o, t, hidden=H, sigma=SIGMA, clip=1.0, seed=SEED, generation=GEN, member_offset=off,
                            n_local=n, precision=precision, workspace=workspace)

    full = run(0, N_LOCAL, None)
    assert bool(torch.isfinite(full).all()) and bool((full <= 0).all())
    assert torch.unique(full).numel() > N_LOCAL // 2                  # members really differ
    workspaces = (None,) if ws is None else (None, ws)
    if ws is not None:
        assert torch.equal(run(0, N_LOCAL, ws), full)                 # mirrored chunks == regenerated chunks
    for off, n in SHARDS:
        for w in workspaces:
            part = run(off, n, w)
            assert torch.equal(part, full[off:off + n]), (off, n, w is not None)
    np.testing.assert_array_equal(run(0, N_LOCAL, None).cpu().numpy(), full.cpu().numpy())   # run to run
