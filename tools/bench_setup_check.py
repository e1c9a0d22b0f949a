"""The proving-key check (b2g_setup_check, Groth16.verify_proving_key) against the rebuild recipe it replaces.

For each circuit kind (chain, circomlike) and --sizes power, under CircomReduction, on one ceremony of the largest power made
by fixed-base products: a key from generate_parameters_from_powers_of_tau with one contribution, then
  check   Groth16.verify_proving_key(circuit, powers, key)
  recipe  generate_parameters_from_powers_of_tau again, the fields a contribution leaves alone compared on the host, then
          Groth16.verify_contribution(rebuilt, key)
on the honest key and on a forged one (one used b_g2_query point negated).  Both arms must give the same verdict on both keys.  The
arms alternate, and each reports the best of --reps calls on the honest key.  --check-only sizes time the check alone (the
recipe's key at those sizes is the setup's cost twice over).  With --profile, one check at the largest --sizes power runs
once more under torch.profiler and its device time is split by stage.  The card name and power limit are read in the same
command.

    python tools/bench_setup_check.py [--sizes 14,16,18,20] [--check-only 22] [--reps 3] [--profile]
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_ptau_check import alternate, ceremony  # noqa: E402
from bench_verify import gpu_label  # noqa: E402
from circom_compat_b200 import Context, Groth16, ProvingKey, synth  # noqa: E402
from circom_compat_b200.zkey import Q_MOD, R_MOD  # noqa: E402

FIXED = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query', 'b_g2_query')


def recipe(ctx, circ, cer, pk):
    rebuilt = Groth16.generate_parameters_from_powers_of_tau(circ, cer, ctx)
    for name in FIXED:
        a, b = np.ascontiguousarray(getattr(rebuilt, name)), np.ascontiguousarray(getattr(pk, name))
        if a.shape != b.shape or a.tobytes() != b.tobytes():
            return False
    return Groth16.verify_contribution(rebuilt, pk, ctx)


def forged(pk):
    b2 = np.array(pk.b_g2_query, copy=True)
    i = int(np.flatnonzero(b2.any(axis=1))[0])                       # a used column: an unused one's point is infinity
    ys = [(Q_MOD - int.from_bytes(b2[i, 8 + 4 * k:12 + 4 * k].tobytes(), 'little')) % Q_MOD for k in range(2)]
    b2[i, 8:] = np.frombuffer(b''.join(y.to_bytes(32, 'little') for y in ys), dtype='<u8')
    fields = {k: getattr(pk, k) for k in ('n_vars', 'n_public', 'domain_size', 'alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2',
                                          'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query', 'l_query', 'h_query')}
    return ProvingKey(b_g2_query=b2, **fields)


def circuit(kind, k):
    return synth.chain_circuit(1 << k) if kind == 'chain' else synth.circomlike_circuit(k)[0]


def profile(ctx, circ, cer, pk):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        assert Groth16.verify_proving_key(circ, cer, pk, ctx=ctx)
        torch.cuda.synchronize()
    split = {'h2d_copy_ms': 0.0, 'point_rules_ms': 0.0, 'g1_sums_and_digit_sort_ms': 0.0, 'g2_sums_ms': 0.0,
             'scalars_ms': 0.0, 'verdict_ms': 0.0, 'other_ms': 0.0}
    for e in p.key_averages():
        us = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0)
        name = e.key
        if 'HtoD' in name:
            key = 'h2d_copy_ms'
        elif 'points_curve' in name or 'g2_subgroup' in name:
            key = 'point_rules_ms'
        elif 'verdict' in name:
            key = 'verdict_ms'
        elif 'Fq2' in name or 'accumulate_g2' in name:
            key = 'g2_sums_ms'
        elif 'msm_' in name or 'powers_' in name:
            key = 'g1_sums_and_digit_sort_ms'
        elif 'check_' in name or 'ntt' in name or 'cub' in name or 'Reduce' in name or 'bitrev' in name:
            key = 'scalars_ms'
        else:
            key = 'other_ms'
        split[key] += us / 1000.0
    return {k: round(v, 2) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='14,16,18,20')
    ap.add_argument('--check-only', default='')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--profile', action='store_true')
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(',') if x]
    only = [int(x) for x in args.check_only.split(',') if x]
    print(json.dumps({'gpu': gpu_label()}), flush=True)
    ctx = Context(0)
    rng = random.Random(0x5E7C)
    cer = ceremony(ctx, max(sizes + only), *(rng.randrange(1, R_MOD) for _ in range(3)))
    for k in sizes + only:
        for kind in ('chain', 'circomlike'):
            circ = circuit(kind, k)
            pk = Groth16.contribute(Groth16.generate_parameters_from_powers_of_tau(circ, cer, ctx), random.Random(k), ctx)
            bad = forged(pk)
            row = {'circuit': kind, 'log_n': k}
            if k in only:
                res = alternate(args.reps, {'check': lambda: Groth16.verify_proving_key(circ, cer, pk, ctx=ctx)})
                if not res['check'][0] or Groth16.verify_proving_key(circ, cer, bad, ctx=ctx):
                    raise SystemExit(f'wrong verdict: {kind} 2^{k}')
                row.update(check_s=round(res['check'][1], 4), recipe_s='not run')
            else:
                res = alternate(args.reps, {'check': lambda: Groth16.verify_proving_key(circ, cer, pk, ctx=ctx),
                                            'recipe': lambda: recipe(ctx, circ, cer, pk)})
                verdicts = {'honest': (bool(res['check'][0]), bool(res['recipe'][0])),
                            'forged': (bool(Groth16.verify_proving_key(circ, cer, bad, ctx=ctx)), bool(recipe(ctx, circ, cer, bad)))}
                if verdicts != {'honest': (True, True), 'forged': (False, False)}:
                    raise SystemExit(f'verdicts differ: {kind} 2^{k}: {verdicts}')
                row.update(check_s=round(res['check'][1], 4), recipe_s=round(res['recipe'][1], 4),
                           speedup=round(res['recipe'][1] / res['check'][1], 2), same_verdicts=True)
            print(json.dumps(row), flush=True)
            if args.profile and k == max(sizes) and kind == 'chain':
                print(json.dumps({'profile': f'chain 2^{k}', **profile(ctx, circ, cer, pk)}), flush=True)
            del circ, pk, bad
    ctx.close()


if __name__ == '__main__':
    main()
