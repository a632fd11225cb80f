"""Novelty-search sweeps' kernels compile clean.  ptxas -v: the five BcSweepArgs instantiations of
rollout_pendulum_kernel (des_envs_bc_sweep.cu) spill nothing and take 64, 79, 121, 141 and 167 registers at H = 16, 32,
64, 96 and 128.  Their twins take 72, 71, 121, 137 and 167 (BcArgs) and 72, 72, 119, 139 and 167 (SweepArgs), so the
larger twin's allocation (8-register granules) is 72, 72, 128, 144 and 168.  The sweep kernel stays within it everywhere
but H = 32, where it takes one granule more (80 allocated against 72): a deviation.  At H = 32 a CTA holds about 8 KB of
shared memory, so an SM fits 28 of them by shared memory, and 80 x 32 registers per CTA lowers that to 25.  The counts
are ceilings: nvcc 12.9 does not schedule this kernel template the same way every time.  Each touches local memory
exactly where its twins do (the frame of the fp64 sincos argument reduction).  des_novelty_runs' kernels and the
per-run blend spill nothing, have no stack frame, and their SASS has no local loads or stores.

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_novelty import _ptxas
from test_sass_runs import LIB, _tool

BC_SWEEP = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb0ENS_11BcSweepArgsEEEvT1_')
BC_SWEEP_REGISTERS = {1: 72, 2: 80, 4: 128, 6: 144, 8: 168}      # R = H/16: ceilings (the docstring)
NOVELTY_RUNS = re.compile(r'_ZN3des19novelty_runs_kernelILi(\d+)EEEvPfPKflS3_liiij')
BLEND_RUNS = '_ZN3des20ns_blend_runs_kernelEPfPKfllPK6float2'


def test_behaviour_sweep_instantiations_keep_their_registers_and_spill_nothing(tmp_path):
    seen = set()
    for name, rep in _ptxas('des_envs_bc_sweep.cu', tmp_path).items():
        m = BC_SWEEP.search(name)
        assert m, name                                      # the unit compiles the behaviour sweep kernels only
        seen.add(int(m.group(1)))
        assert rep['spill'] == 0 and rep['registers'] <= BC_SWEEP_REGISTERS[int(m.group(1))], (name, rep)
    assert seen == set(BC_SWEEP_REGISTERS)


def test_novelty_runs_and_blend_kernels_have_no_stack_and_spill_nothing(tmp_path):
    report = _ptxas('des_novelty.cu', tmp_path)
    assert {int(NOVELTY_RUNS.search(n).group(1)) for n in report if NOVELTY_RUNS.search(n)} == {8, 16, 32}
    assert BLEND_RUNS in report
    for name, rep in report.items():
        assert rep['spill'] == 0 and rep['stack'] == 0, (name, rep)


def test_local_memory_of_the_novelty_sweep_sass():
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
    for R in BC_SWEEP_REGISTERS:
        bc = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_6BcArgsEEEvT1_' % R]
        sweep = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_9SweepArgsEEEvT1_' % R]
        both = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_11BcSweepArgsEEEvT1_' % R]
        assert bc and sweep and len(both) in (len(bc), len(sweep)), (R, bc, sweep, both)
    kernels = [name for name in local if NOVELTY_RUNS.search(name)] + [BLEND_RUNS]
    assert len(kernels) == 4 and all(local[name] == [] for name in kernels)
