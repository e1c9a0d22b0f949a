"""The ceremony check (b2g_powers_check, Groth16.verify_powers_of_tau) and its tableless streamed MSM (b2g_powers_msm).

1. The whole check on an honest ceremony at each --sizes power, as the prefix of one ceremony of the largest power made by
   fixed-base products: from host arrays (Powers.prefix(copy=True)) and from a freshly written .ptau read through its memory
   map.  The file was just written, so its pages are in the page cache: a cold read from disk is not measured.  The two arms
   alternate, and each reports the best of --reps calls.  Host-to-device bytes and their rate over the whole call are listed.
2. With --profile, the largest size once more under torch.profiler, its device time split into the host-to-device copies,
   the point rules, the G1 sums (with the digit sort both groups share), the G2 sum and the verdict.
3. b2g_powers_msm against b2g_msm_g1 / g2 on the same bases and the explicit scalars rho^i (--msm-g1, --msm-g2 sizes), table
   build included since the bases are used once; results compared bit for bit; alternating, best of --reps.
The card name and power limit are read in the same command.

    python tools/bench_ptau_check.py [--sizes 16,18,20,22] [--reps 3] [--profile] [--msm-g1 20,22,24] [--msm-g2 20,22]
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from bench_verify import gpu_label  # noqa: E402
from circom_compat_b200 import Context, Groth16, Powers, read_ptau  # noqa: E402
from circom_compat_b200.zkey import R_MOD  # noqa: E402
import ptau_model  # noqa: E402


def scalars(vals) -> np.ndarray:
    return np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in vals), dtype='<u8').reshape(-1, 4)


def ceremony(ctx, power, tau, alpha, beta):
    n = 1 << power
    t = [1] * (2 * n - 1)
    for i in range(1, 2 * n - 1):
        t[i] = t[i - 1] * tau % R_MOD
    return Powers(power, power, ctx.fixed_base_g1(scalars(t)), ctx.fixed_base_g2(scalars(t[:n])),
                  ctx.fixed_base_g1(scalars([alpha * x % R_MOD for x in t[:n]])),
                  ctx.fixed_base_g1(scalars([beta * x % R_MOD for x in t[:n]])), ctx.fixed_base_g2(scalars([beta])))


def alternate(reps, arms):
    """{name: (last result, best seconds)}, the arms run in turn"""
    best = {}
    for _ in range(reps):
        for name, fn in arms.items():
            t0 = time.perf_counter()
            out = fn()
            dt = time.perf_counter() - t0
            best[name] = (out, min(dt, best.get(name, (None, dt))[1]))
    return best


def profile(ctx, pw, k):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        assert Groth16.verify_powers_of_tau(pw, k, ctx)
        torch.cuda.synchronize()
    split = {'h2d_copy_ms': 0.0, 'point_rules_ms': 0.0, 'g1_sums_and_digit_sort_ms': 0.0, 'g2_sum_ms': 0.0, 'verdict_ms': 0.0,
             'other_ms': 0.0}
    for e in p.key_averages():
        us = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0)
        name = e.key
        if 'HtoD' in name:
            key = 'h2d_copy_ms'
        elif 'powers_rules' in name or 'g2_subgroup' in name:
            key = 'point_rules_ms'
        elif 'verdict' in name:
            key = 'verdict_ms'
        elif 'Fq2' in name or 'accumulate_g2' in name:
            key = 'g2_sum_ms'
        elif 'msm_' in name or 'powers_' in name:
            key = 'g1_sums_and_digit_sort_ms'
        else:
            key = 'other_ms'
        split[key] += us / 1000.0
    return {k: round(v, 2) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='16,18,20,22')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--profile', action='store_true')
    ap.add_argument('--msm-g1', default='20,22,24')
    ap.add_argument('--msm-g2', default='20,22')
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(',') if x]
    print(json.dumps({'gpu': gpu_label()}), flush=True)
    ctx = Context(0)
    rng = random.Random(0x9742)
    if sizes:
        top = max(sizes)
        cer = ceremony(ctx, top, *(rng.randrange(1, R_MOD) for _ in range(3)))
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, 'pot.ptau')
            with open(path, 'wb') as f:
                f.write(ptau_model.write_ptau(top, cer.tau_g1, cer.tau_g2, cer.alpha_tau_g1, cer.beta_tau_g1, cer.beta_g2))
            for k in sizes:
                host = cer.prefix(k, copy=True)
                mapped = read_ptau(path)
                res = alternate(args.reps, {'host': lambda: Groth16.verify_powers_of_tau(host, k, ctx),
                                            'mmap': lambda: Groth16.verify_powers_of_tau(mapped, k, ctx)})
                if not all(r for r, _ in res.values()):
                    raise SystemExit(f'honest ceremony refused at 2^{k}')
                n = 1 << k
                h2d = (2 * n - 1) * 64 + n * 128 + 2 * n * 64 + 128
                print(json.dumps({'log_n': k, 'points': 5 * n, 'h2d_bytes': h2d, 'host_arrays_s': round(res['host'][1], 4),
                                  'mmap_warm_cache_s': round(res['mmap'][1], 4),
                                  'h2d_rate_over_call_GBps': round(h2d / res['host'][1] / 1e9, 2)}), flush=True)
                del host, mapped
            if args.profile:
                print(json.dumps({'profile': f'2^{top} host arrays', **profile(ctx, cer.prefix(top, copy=True), top)}), flush=True)
        del cer
    for g2, spec in ((False, args.msm_g1), (True, args.msm_g2)):
        for k in [int(x) for x in spec.split(',') if x]:
            n = 1 << k
            fb = ctx.fixed_base_g2 if g2 else ctx.fixed_base_g1
            base = fb(scalars([rng.randrange(1, R_MOD) for _ in range(4096)]))
            pts = np.tile(base, (n // 4096, 1))
            rho = rng.randrange(2, R_MOD)
            pw, x = [], 1
            for _ in range(n):
                pw.append(x)
                x = x * rho % R_MOD
            sc = scalars(pw)
            del pw
            msm = ctx.msm_g2 if g2 else ctx.msm_g1
            res = alternate(args.reps, {'powers_msm': lambda: ctx.powers_msm(pts, rho, g2=g2), 'table_msm': lambda: msm(pts, sc)})
            if res['powers_msm'][0].tobytes() != res['table_msm'][0].tobytes():
                raise SystemExit(f"MSMs differ: {'G2' if g2 else 'G1'} 2^{k}")
            print(json.dumps({'msm': 'G2' if g2 else 'G1', 'log_n': k, 'powers_msm_s': round(res['powers_msm'][1], 4),
                              'table_msm_with_table_build_s': round(res['table_msm'][1], 4), 'identical': True}), flush=True)
            del pts, sc
    ctx.close()


if __name__ == '__main__':
    main()
