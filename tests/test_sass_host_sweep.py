"""The kernels of host-stepped sweeps compile like the single-population kernels they extend.  ptxas -v: the sweep
instantiations of policy_act_kernel (parameter block ActSweepArgs) take 32, 32, 35, 44 and 43 registers at H = 16, 32,
64, 96, 128, against 32, 32, 35, 43 and 32 for their ActArgs twins.  The rise at H = 96 costs nothing: registers are
allocated in steps of 8 per thread, so 43 and 44 both take 48.  The rise at H = 128 (the run's key set-up and statistics
row) is intended: a CTA of 128 threads then holds 6144 registers, while its ~100 KB of shared memory (d0 = 24, A = 4)
already limits an SM to 2 CTAs, so it costs no occupancy either.  perturb_sweep_kernel keeps
noise_rows_kernel<true>'s 30 registers although it sets up its round keys from the run's seed.  Nothing spills.
cuobjdump -sass of the built library: none of them accesses local memory.

The sweep instantiations of policy_act_kernel live in des_act_sweep.cu: compiled in des_act.cu beside the ActArgs ones,
they changed ptxas's schedule of policy_act_kernel<64, ActArgs>.

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import subprocess

import pytest

from test_sass_runs import CSRC, LIB, _tool

ACT = re.compile(r'_ZN3des17policy_act_kernelILi(\d+)ENS_(7ActArgs|12ActSweepArgs)EEEvT0_')
SWEEP_REGISTERS = {16: 32, 32: 32, 64: 35, 96: 44, 128: 43}      # see the module docstring
TWIN_REGISTERS = {16: 32, 32: 32, 64: 35, 96: 43, 128: 32}
PERTURB, PERTURB_TWIN = 'perturb_sweep_kernel', 'noise_rows_kernelILb1E'


@pytest.fixture(scope='module')
def report(tmp_path_factory):
    from distributedes_b200.build import NVCC_FLAGS
    nvcc = _tool('nvcc')
    if nvcc is None:
        pytest.skip('nvcc not found')
    out, tmp = {}, tmp_path_factory.mktemp('ptxas')
    for src in ('des_act.cu', 'des_act_sweep.cu', 'des_noise.cu'):
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


def test_policy_act_sweep_instantiations_keep_their_registers_and_spill_nothing(report):
    seen = {}
    for name, rep in report.items():
        m = ACT.search(name)
        if m:
            H, args = int(m.group(1)), m.group(2)
            seen.setdefault(args, set()).add(H)
            want = (SWEEP_REGISTERS if args == '12ActSweepArgs' else TWIN_REGISTERS)[H]
            assert rep['spill'] == 0 and rep['registers'] == want, (name, rep)
            if H != 128:                                                       # the intended exception
                assert -(-rep['registers'] // 8) == -(-TWIN_REGISTERS[H] // 8), (name, rep)    # the twin's allocation
    assert seen == {'7ActArgs': set(TWIN_REGISTERS), '12ActSweepArgs': set(SWEEP_REGISTERS)}


def test_perturb_sweep_kernel_keeps_its_twins_registers(report):
    (rep,) = [r for n, r in report.items() if PERTURB in n]
    (twin,) = [r for n, r in report.items() if PERTURB_TWIN in n]
    assert rep['spill'] == 0 and rep['registers'] == twin['registers'] == 30, (rep, twin)


def test_no_host_sweep_kernel_touches_local_memory():
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
    names = [n for n in local if PERTURB in n or '12ActSweepArgs' in n]
    assert len(names) == 6, names
    for name in names:
        assert not local[name], (name, local[name])
