"""The mirrored-sampling instantiations of the tensor-core forward (eval_tc_mirrored_kernel: the body of eval_tc_kernel
with the producers' kMirror flag set) keep the CTA-scope hand-off that tests/test_sass_handoff.py checks on the plain
ones: no GPU-scope fence, an L1 invalidation only after the cluster barrier at kernel start, bulk copies of the peer's half
in 2-CTA clusters.  Every (H, precision, cluster, action bound) has a mirrored instantiation.

Reads the SASS of the built library with cuobjdump; skips where either is missing."""
import os
import re
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(REPO, 'distributedes_b200', 'libdes_b200.so')
KERNEL = re.compile(r'_ZN3des23eval_tc_mirrored_kernelILi(\d+)ELb([01])ELi([12])ELi(\d+)EEEvNS_6TcArgsE')


@pytest.fixture(scope='module')
def mirrored_sass():
    tool = shutil.which('cuobjdump') or ('/usr/local/cuda/bin/cuobjdump'
                                         if os.path.exists('/usr/local/cuda/bin/cuobjdump') else None)
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


def test_every_mirrored_instantiation_keeps_the_cta_scope_hand_off(mirrored_sass):
    assert sorted(mirrored_sass) == sorted((H, x3, CL, NA) for H in (64, 128, 256) for x3 in (False, True)
                                           for CL in (1, 2) for NA in (4, 8))
    for key, ins in mirrored_sass.items():
        _, _, CL, _ = key
        assert not [i for i in ins if 'MEMBAR.ALL.GPU' in i], key
        cctl = [k for k, i in enumerate(ins) if 'CCTL.IVALL' in i]
        waits = [k for k, i in enumerate(ins) if 'UCGABAR_WAIT' in i]
        assert len(waits) == (1 if CL == 2 else 0) and all(k - 1 in waits for k in cctl), key
        assert (sum('UBLKCP' in i for i in ins) > 0) == (CL == 2), key
        assert not [i for i in ins if i.split()[0] in ('STL', 'LDL') or ' STL' in i or ' LDL' in i], key   # no spills
