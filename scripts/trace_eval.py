"""Phase trace of the tensor-core policy forward (eval_tc_kernel) at the headline shape.

Builds the library variant with -DDES_EVAL_TRACE (scripts/build_variant.sh trace des_eval_tc.cu -DDES_EVAL_TRACE), runs
one NES generation of scripts/profile_gen.py with it (DES_LIB_PATH), and prints each role's clock64() totals per warp
and per member: barrier waits, MMA issue -> wgmma_wait, fences and arrivals, epilogues, weight generation, the rest.

    python scripts/trace_eval.py [--lib PATH] [--pop 65536] [--hidden 256] [--precision f16x3]

--lib runs an already built trace library instead of building one (for instance an older kernel's, to compare).
"""
import argparse
import collections
import os
import re
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ['wait', 'mma', 'sync', 'epi', 'gen', 'other', 'total']
LINE = re.compile(r'DES_TRACE cta=(\d+) warp=(\d+) role=(\w+) members=(\d+) ' +
                  ' '.join(r'%s=(\d+)' % p for p in PHASES))


def parse(text):
    """{(cta, role): [per-warp dict]} from the kernel's printf lines"""
    out = collections.defaultdict(list)
    for m in LINE.finditer(text):
        cta, warp, role, members = int(m.group(1)), int(m.group(2)), m.group(3), int(m.group(4))
        d = {p: int(m.group(5 + k)) for k, p in enumerate(PHASES)}
        d.update(warp=warp, members=members)
        out[(cta, role)].append(d)
    return out


def report(rows):
    print('kilocycles per member and warp (mean over the role\'s warps)')
    print('%-5s %-9s %7s ' % ('cta', 'role', 'members') + ' '.join('%8s' % p for p in PHASES))
    for (cta, role), warps in sorted(rows.items()):
        members = warps[0]['members']
        mean = {p: sum(w[p] for w in warps) / len(warps) / max(members, 1) / 1e3 for p in PHASES}
        print('%-5d %-9s %7d ' % (cta, role, members) + ' '.join('%8.2f' % mean[p] for p in PHASES))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--lib', help='trace build of the library to run (default: build it)')
    ap.add_argument('--pop', type=int, default=65536)
    ap.add_argument('--hidden', type=int, default=256)
    ap.add_argument('--precision', default='f16x3')
    args = ap.parse_args()
    lib = args.lib
    if lib is None:
        r = subprocess.run(['bash', os.path.join(REPO, 'scripts', 'build_variant.sh'), 'trace', 'des_eval_tc.cu',
                            '-DDES_EVAL_TRACE'], cwd=REPO, capture_output=True, text=True, check=True)
        lib = os.path.join(REPO, r.stdout.strip().splitlines()[-1])
    env = dict(os.environ, DES_LIB_PATH=os.path.abspath(lib))
    r = subprocess.run([sys.executable, os.path.join(REPO, 'scripts', 'profile_gen.py'), str(args.pop),
                        str(args.hidden), args.precision, '1'], env=env, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        sys.exit(r.returncode)
    rows = parse(r.stdout)
    if not rows:
        sys.exit('no DES_TRACE lines: is %s a -DDES_EVAL_TRACE build?' % lib)
    print('library %s, pop %d, H %d, %s' % (lib, args.pop, args.hidden, args.precision))
    report(rows)


if __name__ == '__main__':
    main()
