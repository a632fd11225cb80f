"""The genetic-algorithm sweep kernels compile like the kernels they extend.  ptxas -v: the five GaSweepArgs
instantiations of rollout_pendulum_kernel (des_envs_ga_sweep.cu) took 72, 72, 95, 139 and 167 registers at H = 16, 32,
64, 96 and 128, against 72, 71, 121, 127 and 167 for their GaArgs twins and 72, 72, 119, 139 and 167 for the SweepArgs
kernels of NES sweeps.  Registers are allocated in steps of 8 per thread, so H = 16, 32, 64 and 128 stay within their
GaArgs twin's allocation.  At H = 96 the kernel takes what the SweepArgs kernel takes, two steps above its GaArgs twin:
the round keys set up from the run's seed live in registers rather than in the parameter bank, as in every sweep kernel.
An H = 96 CTA needs 46 KB of shared memory, so shared memory, not registers, bounds its occupancy (four CTAs per SM
either way).  The ceilings below are the larger of the two twins' allocations, not pins: nvcc 12.9 does not compile this
kernel template the same way every time (test_sass_record.py).  None spills, and each touches local memory exactly where
its GaArgs twin does (the 40-byte frame of the fp64 sincos argument reduction).  The table kernels of des_ga_sweep.cu
take at most 40 registers and have no stack frame.

The GaSweepArgs instantiations live in des_envs_ga_sweep.cu and the table kernels in des_ga_sweep.cu, so that
des_envs.cu, des_envs_sweep.cu, des_envs_ga.cu and des_ga.cu compile exactly the kernels they did.

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_ga import _ptxas
from test_sass_runs import LIB, _tool

GA_SWEEP = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb0ENS_11GaSweepArgsEEEvT1_')
GA_SWEEP_REGISTERS = {1: 72, 2: 72, 4: 128, 6: 144, 8: 168}          # R = H/16: ceilings
TABLE_KERNELS = {'ga_rows_sweep_kernel': 40, 'ga_negate_runs_kernel': 16, 'ga_scatter_runs_kernel': 16}


def test_ga_sweep_rollout_instantiations_keep_their_registers_and_spill_nothing(tmp_path):
    seen = set()
    for name, rep in _ptxas('des_envs_ga_sweep.cu', tmp_path).items():
        m = GA_SWEEP.search(name)
        assert m, name                                      # the unit compiles the GA sweep kernels only
        R = int(m.group(1))
        seen.add(R)
        assert rep['spill'] == 0 and rep['registers'] <= GA_SWEEP_REGISTERS[R], (name, rep)
    assert seen == set(GA_SWEEP_REGISTERS)


def test_sweep_table_kernels_have_no_stack_frame(tmp_path):
    rep = _ptxas('des_ga_sweep.cu', tmp_path)
    assert len(rep) == len(TABLE_KERNELS)
    for name, r in rep.items():
        short = next(k for k in TABLE_KERNELS if k in name)
        assert r['spill'] == 0 and r['frame'] == 0 and r['registers'] <= TABLE_KERNELS[short], (name, r)


def test_local_memory_of_the_ga_sweep_sass():
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
    for R in GA_SWEEP_REGISTERS:
        twin = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_6GaArgsEEEvT1_' % R]
        sweep = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_11GaSweepArgsEEEvT1_' % R]
        assert twin and len(sweep) == len(twin), (R, twin, sweep)
    for name, ins in local.items():
        if any(k in name for k in TABLE_KERNELS):
            assert not ins, (name, ins)
