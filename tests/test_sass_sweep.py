"""The sweep instantiations compile like the run-batched kernels they extend.  ptxas -v: the sweep rollout kernels
(parameter block SweepArgs) take 72, 72, 119, 139 and 167 registers at H = 16, 32, 64, 96, 128, against 72, 71, 121, 141
and 167 for their RunArgs twins.  The one rise, at H = 32, is intended: registers are allocated in steps of 8 per thread,
so 71 and 72 both take 72 and the per-CTA key set-up from the run's seed costs no occupancy.  grad_chunk_sweep_kernel
keeps grad_chunk_kernel<false, true>'s 32 registers although its round keys live in registers rather than in the
parameter bank, and apply_sweep_kernel keeps apply_runs_kernel's 40.  Nothing spills.
cuobjdump -sass of the built library: the sweep grad and apply kernels have no local-memory access at all, and a sweep
rollout kernel touches local memory exactly where its RunArgs twin does (the 40-byte frame of the fp64 sincos argument
reduction).

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_runs import LIB, RUN_REGISTERS, _tool, ptxas_report  # noqa: F401

SWEEP_REGISTERS = {1: 72, 2: 72, 4: 119, 6: 139, 8: 167}        # R = H/16 -> registers; see the module docstring
SWEEP_ROLLOUT = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb0ENS_9SweepArgsEEEvT1_')
KERNELS = {'grad_chunk_sweep_kernel': 32, 'apply_sweep_kernel': 40}
TWINS = {'grad_chunk_sweep_kernel': 'grad_chunk_kernelILb0ELb1E', 'apply_sweep_kernel': 'apply_runs_kernel'}


def test_sweep_rollout_instantiations_keep_their_registers_and_spill_nothing(ptxas_report):  # noqa: F811
    seen = set()
    for name, rep in ptxas_report.items():
        m = SWEEP_ROLLOUT.search(name)
        if m:
            R = int(m.group(1))
            seen.add(R)
            assert rep['spill'] == 0, (name, rep)
            assert rep['registers'] == SWEEP_REGISTERS[R], (name, rep)
            assert rep['registers'] <= -(-RUN_REGISTERS[R] // 8) * 8, (name, rep)     # the twin's allocation
    assert seen == set(SWEEP_REGISTERS)


def test_sweep_grad_and_apply_kernels_keep_their_twins_registers(ptxas_report):  # noqa: F811
    for tag, registers in KERNELS.items():
        (rep,) = [r for n, r in ptxas_report.items() if tag in n]
        (twin,) = [r for n, r in ptxas_report.items() if TWINS[tag] in n]
        assert rep['spill'] == 0 and rep['registers'] == registers == twin['registers'], (tag, rep, twin)


def test_local_memory_of_the_sweep_sass():
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
    for tag in KERNELS:
        (name,) = [n for n in local if tag in n]
        assert not local[name], (name, local[name])
    for R in SWEEP_REGISTERS:
        runs = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_7RunArgsEEEvT1_' % R]
        sweep = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_9SweepArgsEEEvT1_' % R]
        assert runs and len(sweep) == len(runs), (R, runs, sweep)
