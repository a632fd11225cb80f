"""Time NES generations with plain and mirrored sampling, alternated in one process: ms per generation, the forward kernel
(des_nes_eval / des_nes_eval_mirrored) and the fitness x noise reduction (des_nes_grad_partial[_mirrored]).

Every generation runs eager, with a 256 MiB memset before it (outside the events) so it starts with a cold L2, as bench.py
does; CUDA events bracket the whole generation, the evaluation and the reduction.  Rounds alternate plain and mirrored
engines of the same shape; each value is the median over the rounds' per-generation means.  The card's name and power
limit are read with nvidia-smi in the same run.

    python scripts/time_mirrored.py [--steps 10] [--rounds 3] [--out time_mirrored.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np      # noqa: E402
import torch            # noqa: E402
from distributedes_b200.engine import NESEngine       # noqa: E402
from oracle import nes_oracle as orc                   # noqa: E402

SHAPES = [(65536, 256, 256, 'f16x3'), (65536, 256, 256, 'f16'), (16384, 256, 256, 'f16x3')]     # pop, H, T, precision


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = 'nvidia-smi unavailable (%s)' % e
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q)


def engine(pop, H, T, precision, mirrored):
    d0, A = 24, 4
    obs, target = orc.synthetic_tape(T, d0, A)
    return NESEngine(state_dim=d0, hidden=H, action_dim=A, pop_size=pop, theta0=orc.synthetic_theta(d0, H, A), obs=obs,
                     target=target, sigma=0.1, learning_rate=0.1, seed=3, precision=precision, device='cuda:0',
                     mirrored=mirrored)


def time_engine(eng, steps, flush):
    """Mean ms per generation, per forward kernel and per reduction over `steps` eager generations."""
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(6)] for _ in range(steps)]
    for s in range(steps):
        flush.zero_()
        e = ev[s]
        e[0].record()
        e[1].record()
        eng.evaluate()
        e[2].record()
        eng.k.centered_rank(eng.fitness_all, eng.offset, eng.n_local, workspace=eng.rank_ws, out=eng.shaped)
        e[3].record()
        grad = eng.k.nes_grad_partial_mirrored if eng.mirrored else eng.k.nes_grad_partial
        grad(eng.shaped, eng.P, seed=eng.seed, state=eng.state, member_offset=eng.offset, workspace=eng.grad_ws,
             out=eng.partial)
        e[4].record()
        eng.apply()
        e[5].record()
        eng.generation_index += 1
    torch.cuda.synchronize()
    gen = np.mean([e[0].elapsed_time(e[5]) for e in ev])
    fwd = np.mean([e[1].elapsed_time(e[2]) for e in ev])
    red = np.mean([e[3].elapsed_time(e[4]) for e in ev])
    return gen, fwd, red


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda:0')       # > 50 MB L2 (H100)
    result = dict(card=card(), steps=a.steps, rounds=a.rounds, shapes=[])
    for pop, H, T, precision in SHAPES:
        engs = {m: engine(pop, H, T, precision, m) for m in (False, True)}
        for e in engs.values():
            time_engine(e, 2, flush)                                           # warm-up: module loading, first launches
        runs = {False: [], True: []}
        for _ in range(a.rounds):
            for m in (False, True):
                runs[m].append(time_engine(engs[m], a.steps, flush))
        row = dict(pop=pop, hidden=H, tape_len=T, precision=precision)
        for m, name in ((False, 'plain'), (True, 'mirrored')):
            r = np.asarray(runs[m])
            row[name] = dict(ms_per_generation=float(np.median(r[:, 0])), forward_ms=float(np.median(r[:, 1])),
                             reduction_ms=float(np.median(r[:, 2])), rounds=r.round(4).tolist())
        row['reduction_ratio'] = row['mirrored']['reduction_ms'] / row['plain']['reduction_ms']
        result['shapes'].append(row)
        print(json.dumps(row), flush=True)
        del engs
        torch.cuda.empty_cache()
    result['card_after'] = card()
    print(json.dumps(result['card']))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
