"""The genetic algorithm's novelty-search kernels compile clean.  ptxas -v: the five GaBcArgs instantiations of
rollout_pendulum_kernel (des_envs_ga_bc.cu) spill nothing and take 72, 71, 121, 137 and 167 registers at H = 16, 32, 64,
96 and 128.  Their twins take 72, 71, 121, 127 and 167 (GaArgs) and 72, 71, 121, 137 and 167 (BcArgs), so the larger
twin's allocation (8-register granules) is 72, 72, 128, 144 and 168, and the kernel stays within it at every width.
Against the GaArgs twin alone it takes one granule more at H = 96 (144 allocated against 128), as the BcArgs kernel does
against RollArgs: shared memory (about 46 KB per CTA at H = 96) already limits an SM to four 32-thread CTAs there, so
occupancy is unchanged.  The counts are ceilings: nvcc 12.9 does not schedule this kernel template the same way every
time.  Each touches local memory exactly where its twins do (the frame of the fp64 sincos argument reduction).
des_ns_ga_order launches only existing kernels (ga_negate_kernel, des_ns_shape's, des_centered_rank's,
ga_scatter_kernel); the two of des_ga.cu have no stack frame and spill nothing.

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_novelty import _ptxas
from test_sass_runs import LIB, _tool

GA_BC = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb0ENS_8GaBcArgsEEEvT1_')
GA_BC_REGISTERS = {1: 72, 2: 72, 4: 128, 6: 144, 8: 168}      # R = H/16: ceilings (the docstring)
ORDER = ('_ZN3des16ga_negate_kernelEPfPKfl', '_ZN3des17ga_scatter_kernelEPiPKill')


def test_ga_behaviour_instantiations_keep_their_registers_and_spill_nothing(tmp_path):
    seen = set()
    for name, rep in _ptxas('des_envs_ga_bc.cu', tmp_path).items():
        m = GA_BC.search(name)
        assert m, name                                      # the unit compiles the GA behaviour kernels only
        seen.add(int(m.group(1)))
        assert rep['spill'] == 0 and rep['registers'] <= GA_BC_REGISTERS[int(m.group(1))], (name, rep)
    assert seen == set(GA_BC_REGISTERS)


def test_order_kernels_have_no_stack_and_spill_nothing(tmp_path):
    report = _ptxas('des_ga.cu', tmp_path)
    for name in ORDER:
        assert name in report, sorted(report)
        assert report[name]['spill'] == 0 and report[name]['stack'] == 0, (name, report[name])


def test_local_memory_of_the_ga_novelty_sass():
    tool = _tool('cuobjdump')
    if tool is None or not os.path.exists(LIB):
        pytest.skip('cuobjdump or the built library missing')
    r = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    local, cur = {}, None
    for line in r.stdout.splitlines():
        if 'Function :' in line:
            cur = line.split('Function :')[1].strip()
            local[cur] = []
        elif cur is not None and re.match(r'\s*/\*[0-9a-f]{4,}\*/', line):
            ins = line.split(';')[0].split('*/', 1)[1].strip()
            if re.search(r'\b(STL|LDL)\b', ins):
                local[cur].append(ins)
    for R in GA_BC_REGISTERS:
        ga = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_6GaArgsEEEvT1_' % R]
        bc = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_6BcArgsEEEvT1_' % R]
        both = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_8GaBcArgsEEEvT1_' % R]
        assert ga and bc and len(both) in (len(ga), len(bc)), (R, ga, bc, both)
    assert all(local[name] == [] for name in ORDER)
