"""The kernels of CMA-ES sweeps compile like the kernels they extend.  ptxas -v: the row-mode sweep rollout kernels
(rollout_pendulum_kernel<R, true, SweepArgs>, des_envs_sweep.cu) take 64, 79, 121, 141 and 167 registers at H = 16, 32,
64, 96, 128, against 72, 71, 121, 127 and 167 for their RollArgs twins.  Two rises, both accepted:
  - H = 96 (141, as the NES run-batched kernel at that width): a CTA's ~46 KB of shared memory already limits an SM to 4
    CTAs of one warp, far below what 141 registers allow.
  - H = 32 (79, allocated as 80): the run's round keys, set up from its seed, live in registers.  A CTA's 7.9 KB of shared
    memory (plus 1 KB the SM reserves) limits an SM to 26 CTAs; 80 registers allow 25, so a full SM holds one CTA in 26
    fewer.  That bites only past 25 x 132 = 3300 rows in flight: the reference's experiment, 10 runs of 64, is 640.
cma_rank_mu_runs_kernel keeps cma_rank_mu_kernel's 64 registers, and noise_sweep_kernel takes 20 against
noise_rows_kernel<false>'s 28.  cma_cov_runs_kernel takes 20 against cma_cov_apply_kernel's 17: both are allocated
as 24.  Nothing spills.  cuobjdump -sass of the built library: none of the new kernels but the rollout ones accesses local
memory, and a row-mode sweep rollout kernel touches it exactly where its RollArgs twin does (the 40-byte frame of the fp64
sincos argument reduction).

The row-mode sweep instantiations live in des_envs_sweep.cu: compiled in des_envs.cu beside the others, they changed
ptxas's schedule of rollout_pendulum_kernel<8, true, RollArgs>.

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_runs import CSRC, LIB, REGISTERS, _tool

ROWS_SWEEP = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb1ENS_9SweepArgsEEEvT1_')
ROWS_SWEEP_REGISTERS = {1: 64, 2: 79, 4: 121, 6: 141, 8: 167}           # R = H/16; see the module docstring
KERNELS = {'cma_rank_mu_runs_kernel': 64, 'cma_cov_runs_kernel': 20, 'noise_sweep_kernel': 20}
TWINS = {'cma_rank_mu_runs_kernel': ('cma_rank_mu_kernel', 64), 'cma_cov_runs_kernel': ('cma_cov_apply_kernel', 17),
         'noise_sweep_kernel': ('noise_rows_kernelILb0E', 28)}


@pytest.fixture(scope='module')
def report(tmp_path_factory):
    from distributedes_b200.build import NVCC_FLAGS
    nvcc = _tool('nvcc')
    if nvcc is None:
        pytest.skip('nvcc not found')
    out, tmp = {}, tmp_path_factory.mktemp('ptxas')
    for src in ('des_envs_sweep.cu', 'des_cma.cu', 'des_noise.cu'):
        r = subprocess.run([nvcc] + NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(CSRC, src), '-o',
                                                  str(tmp / (src + '.o'))], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        cur = None
        for line in r.stderr.splitlines():
            m = re.search(r"Compiling entry function '(\S+)'", line)
            if m:
                cur = m.group(1)
                out[cur] = {}
            m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
            if m and cur:
                out[cur]['spill'] = int(m.group(1)) + int(m.group(2))
            m = re.search(r'Used (\d+) registers', line)
            if m and cur:
                out[cur]['registers'] = int(m.group(1))
    return out


def test_row_mode_sweep_rollout_instantiations_keep_their_registers_and_spill_nothing(report):
    seen = set()
    for name, rep in report.items():
        m = ROWS_SWEEP.search(name)
        if m:
            R = int(m.group(1))
            seen.add(R)
            assert rep['spill'] == 0 and rep['registers'] == ROWS_SWEEP_REGISTERS[R], (name, rep)
            if R not in (2, 6):                                                 # the accepted rises
                assert -(-rep['registers'] // 8) <= -(-REGISTERS[R] // 8), (name, rep)
    assert seen == set(ROWS_SWEEP_REGISTERS)


def test_run_batched_cma_kernels_keep_their_registers_and_spill_nothing(report):
    for tag, registers in KERNELS.items():
        (rep,) = [r for n, r in report.items() if tag in n]
        twin_tag, twin_registers = TWINS[tag]
        (twin,) = [r for n, r in report.items() if twin_tag in n and 'runs' not in n]
        assert rep['spill'] == 0 and rep['registers'] == registers, (tag, rep)
        assert twin['registers'] == twin_registers, (twin_tag, twin)
        assert -(-rep['registers'] // 8) <= -(-twin['registers'] // 8), (tag, rep, twin)


def test_local_memory_of_the_cma_sweep_sass():
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
    for R in ROWS_SWEEP_REGISTERS:
        plain = local['_ZN3des23rollout_pendulum_kernelILi%dELb1ENS_8RollArgsEEEvT1_' % R]
        sweep = local['_ZN3des23rollout_pendulum_kernelILi%dELb1ENS_9SweepArgsEEEvT1_' % R]
        assert plain and len(sweep) == len(plain), (R, plain, sweep)
