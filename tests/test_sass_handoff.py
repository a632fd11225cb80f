"""The tensor-core forward's producer -> consumer hand-off compiles to CTA-scope synchronisation only (no GPU).

Every instantiation of eval_tc_kernel hands its weight tiles over with CTA-scope mbarriers, and a 2-CTA cluster pushes
each CTA's half to its peer with bulk copies (UBLKCP).  A cluster-scope release (mbarrier.arrive.release.cluster,
fence.proxy.async.shared::cluster) compiles to MEMBAR.ALL.GPU and a cluster-scope acquire to CCTL.IVALL, an L1
invalidation: one of either in the per-chunk loop costs the kernel several milliseconds at the headline shape.  The
only CCTL.IVALL allowed is the one after the cluster barrier at kernel start (barrier.cluster.wait always acquires),
which runs once per launch.

Reads the SASS of the built library with cuobjdump; skips where either is missing.
"""
import os
import re
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(REPO, 'distributedes_b200', 'libdes_b200.so')
KERNEL = re.compile(r'_ZN3des14eval_tc_kernelILi(\d+)ELb([01])ELi([12])ELi(\d+)EEEvNS_6TcArgsE')


def _cuobjdump():
    tool = shutil.which('cuobjdump')
    if tool is None and os.path.exists('/usr/local/cuda/bin/cuobjdump'):
        tool = '/usr/local/cuda/bin/cuobjdump'
    return tool


@pytest.fixture(scope='module')
def eval_sass():
    """{(H, x3, CL, NA): list of SASS instruction lines} of every eval_tc_kernel instantiation"""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip('cuobjdump not found')
    if not os.path.exists(LIB):
        pytest.skip('library not built')
    r = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    out, cur = {}, None
    for line in r.stdout.splitlines():
        if 'Function :' in line:
            m = KERNEL.search(line)
            cur = (int(m.group(1)), m.group(2) == '1', int(m.group(3)), int(m.group(4))) if m else None
            if cur is not None:
                out[cur] = []
        elif cur is not None and re.match(r'\s*/\*[0-9a-f]{4,}\*/', line):
            out[cur].append(line.split(';')[0].split('*/', 1)[1].strip())
    return out


def test_every_instantiation_found(eval_sass):
    assert sorted(eval_sass) == sorted((H, x3, CL, NA) for H in (64, 128, 256) for x3 in (False, True)
                                       for CL in (1, 2) for NA in (4, 8))


def test_no_gpu_scope_fence(eval_sass):
    for key, ins in eval_sass.items():
        assert not [i for i in ins if 'MEMBAR.ALL.GPU' in i], key


def test_l1_invalidation_only_at_kernel_start(eval_sass):
    for key, ins in eval_sass.items():
        cctl = [k for k, i in enumerate(ins) if 'CCTL.IVALL' in i]
        waits = [k for k, i in enumerate(ins) if 'UCGABAR_WAIT' in i]
        _, _, CL, _ = key
        assert len(waits) == (1 if CL == 2 else 0), key
        assert len(cctl) <= len(waits), key
        assert all(k - 1 in waits for k in cctl), key


def test_clusters_move_the_peer_half_by_bulk_copy(eval_sass):
    for key, ins in eval_sass.items():
        _, _, CL, _ = key
        n = sum('UBLKCP' in i for i in ins)
        assert (n > 0) == (CL == 2), (key, n)
