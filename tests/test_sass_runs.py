"""The run-batched instantiations compile like the single-population kernels they extend.  ptxas -v: every plain
rollout_pendulum_kernel instantiation (parameter block RollArgs) keeps the registers of its width (H = 16, 32, 64, 96, 128:
72, 71, 121, 127, 167), and every instantiation spills nothing.  The run-batched ones (parameter block RunArgs) are
pinned too: the same counts except at H = 96, where the run's theta and statistics rows cost 14 registers (141).  That
exception is intended: at H = 96 a CTA's ~46 KB of shared memory already limits an SM to 4 CTAs of one warp, far below
what 141 registers allow, so the run offset costs no occupancy.  The run-batched rank, grad, apply and statistics kernels
spill nothing either.
cuobjdump -sass of the built library: those four have no local-memory access at all, and a run-batched rollout kernel
touches local memory exactly where its plain twin does (the 40-byte frame of the fp64 sincos argument reduction).

Needs nvcc (and the built library for the SASS); skips where either is missing."""
import os
import re
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, 'distributedes_b200', 'csrc')
LIB = os.path.join(REPO, 'distributedes_b200', 'libdes_b200.so')
REGISTERS = {1: 72, 2: 71, 4: 121, 6: 127, 8: 167}          # R = H/16 -> registers
RUN_REGISTERS = {**REGISTERS, 6: 141}                       # the intended exception: see the module docstring
ROLLOUT = re.compile(r'_ZN3des23rollout_pendulum_kernelILi(\d)ELb([01])ENS_(8RollArgs|7RunArgs)EEEvT1_')
RUNS = ('grad_chunk_kernelILb0ELb1E', 'rank_count_runs_kernel', 'apply_runs_kernel', 'grad_reduce_runs_kernel',
        'stat_part_reduce_runs_kernel', 'obs_stats_merge_totals_runs_kernel')


def _tool(name):
    return shutil.which(name) or next((p for p in ['/usr/local/cuda/bin/' + name] if os.path.exists(p)), None)


@pytest.fixture(scope='module')
def ptxas_report(tmp_path_factory):
    from distributedes_b200.build import NVCC_FLAGS
    nvcc = _tool('nvcc')
    if nvcc is None:
        pytest.skip('nvcc not found')
    out, tmp = {}, tmp_path_factory.mktemp('ptxas')
    for src in ('des_envs.cu', 'des_update.cu', 'des_rank.cu', 'des_obs.cu'):
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


def test_rollout_instantiations_keep_their_registers_and_spill_nothing(ptxas_report):
    seen = set()
    for name, rep in ptxas_report.items():
        m = ROLLOUT.search(name)
        if m:
            R, rows, runs = int(m.group(1)), m.group(2) == '1', m.group(3) == '7RunArgs'
            seen.add((R, rows, runs))
            assert rep['spill'] == 0, (name, rep)
            assert rep['registers'] == (RUN_REGISTERS if runs else REGISTERS)[R], (name, rep)
    assert seen == {(R, rows, False) for R in REGISTERS for rows in (False, True)} | {(R, False, True) for R in REGISTERS}


def test_run_batched_kernels_spill_nothing(ptxas_report):
    for tag in RUNS:
        hits = [rep for name, rep in ptxas_report.items() if tag in name]
        assert len(hits) == 1, tag
        assert hits[0]['spill'] == 0, (tag, hits[0])


def test_local_memory_of_the_run_batched_sass():
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
    for tag in RUNS:
        (name,) = [n for n in local if tag in n]
        assert not local[name], (name, local[name])
    for R in REGISTERS:
        plain = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_8RollArgsEEEvT1_' % R]
        runs = local['_ZN3des23rollout_pendulum_kernelILi%dELb0ENS_7RunArgsEEEvT1_' % R]
        assert plain and len(runs) == len(plain), (R, plain, runs)
