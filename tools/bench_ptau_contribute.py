"""Phase-1 contributions (b2g_powers_contribute) and the per-point product they run (b2g_points_scale).

1. Context.points_scale on 2^20 and 2^22 G1 and G2 points with one random scalar each, in points per second, best of --reps.
2. Groth16.contribute_powers_of_tau at each --powers power on an honest ceremony the script writes to a temporary file (a
   contribution to the new ceremony) and reads back memory-mapped; the output goes to a second file.  Best of --reps.  Power 24
   is added when the host has room for it (--powers can name it explicitly).
3. With --profile DIR, instead: one contribution at the first --powers power under torch.profiler (CUDA activities), the
   kernel table written to DIR/contribute_profile.txt.
The card name and power limit are read in the same command.

    python tools/bench_ptau_contribute.py [--scale 20,22] [--powers 16,18,20,22] [--reps 3] [--profile DIR]
"""
import argparse
import json
import os
import random
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_verify import gpu_label  # noqa: E402
from circom_compat_b200 import Context, Groth16, new_powers_of_tau, read_ptau  # noqa: E402
from circom_compat_b200.zkey import R_MOD  # noqa: E402


def scalars(rng, n):
    distinct = np.frombuffer(b''.join(rng.randrange(R_MOD).to_bytes(32, 'little') for _ in range(min(n, 1 << 16))),
                             dtype='<u8').reshape(-1, 4)
    return np.tile(distinct, ((n + len(distinct) - 1) // len(distinct), 1))[:n].copy()


def bench_scale(ctx, logs, reps):
    rng = random.Random(1)
    for g2 in (False, True):
        fb = ctx.fixed_base_g2 if g2 else ctx.fixed_base_g1
        for lg in logs:
            n = 1 << lg
            base = fb(scalars(rng, 1 << 12))
            pts = np.tile(base, (n // len(base), 1))
            ks = scalars(rng, n)
            ctx.points_scale(pts[:1024], ks[:1024], g2=g2)                  # module load
            best = min(timed(lambda: ctx.points_scale(pts, ks, g2=g2)) for _ in range(reps))
            print(json.dumps({'op': 'points_scale', 'group': 'G2' if g2 else 'G1', 'log_n': lg, 's': round(best, 4),
                              'points_per_s': round(n / best)}), flush=True)


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def honest_file(ctx, power, path):
    rng = random.Random(power)
    Groth16.contribute_powers_of_tau(new_powers_of_tau(power), dst=path, ctx=ctx,
                                     tau=rng.randrange(1, R_MOD), alpha=rng.randrange(1, R_MOD), beta=rng.randrange(1, R_MOD))
    return read_ptau(path)


def host_room(power) -> bool:
    """the input and output files of a contribution at this power, with room to spare, fit in available host memory"""
    need = 2 * ((4 << power) * 64 + (1 << power) * 128) * 2
    try:
        avail = os.sysconf('SC_AVPHYS_PAGES') * os.sysconf('SC_PAGE_SIZE')
    except (ValueError, OSError):
        return False
    return avail > need


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scale', default='20,22')
    ap.add_argument('--powers', default='16,18,20,22')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--profile', default=None)
    args = ap.parse_args()
    sizes = lambda s: [int(x) for x in s.split(',') if x]
    powers = sizes(args.powers)
    ctx = Context(0)
    print(json.dumps({'gpu': gpu_label()}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        if args.profile:
            import torch
            from torch.profiler import ProfilerActivity, profile
            p = powers[0]
            src = honest_file(ctx, p, os.path.join(tmp, 'in.ptau'))
            Groth16.contribute_powers_of_tau(new_powers_of_tau(2), ctx=ctx, tau=2, alpha=3, beta=4)   # module load
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                Groth16.contribute_powers_of_tau(src, dst=os.path.join(tmp, 'out.ptau'), ctx=ctx)
                torch.cuda.synchronize()
            os.makedirs(args.profile, exist_ok=True)
            table = prof.key_averages().table(sort_by='cuda_time_total', row_limit=25)
            with open(os.path.join(args.profile, 'contribute_profile.txt'), 'w') as f:
                f.write(f"power {p}\n{table}\n")
            print(table, flush=True)
            return
        bench_scale(ctx, sizes(args.scale), args.reps)
        if 24 not in powers and host_room(24):
            powers.append(24)
        for p in powers:
            src = honest_file(ctx, p, os.path.join(tmp, 'in.ptau'))
            best = min(timed(lambda: Groth16.contribute_powers_of_tau(src, dst=os.path.join(tmp, 'out.ptau'), ctx=ctx))
                       for _ in range(args.reps))
            g1, g2 = (4 << p) - 1, (1 << p) + 1
            print(json.dumps({'op': 'contribute', 'power': p, 's': round(best, 3), 'g1_points': g1, 'g2_points': g2}), flush=True)
            del src


if __name__ == '__main__':
    main()
