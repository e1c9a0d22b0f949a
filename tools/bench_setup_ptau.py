"""Groth16 setup from a powers-of-tau ceremony (b2g_setup_from_powers), one delta contribution (b2g_delta_update) and its
check (b2g_delta_update_check), with b2g_setup on the same circuit for scale.  Each key from the ceremony is compared byte for
byte with b2g_setup(alpha, beta, 1, 1, tau) before anything is reported.

The ceremony (2^max(sizes) powers of seeded tau, alpha, beta) is made by fixed-base products on the GPU and written as a
.ptau file to a temporary directory; `ptau_read_s` is read_ptau plus copying the prefix the circuit needs out of the memory
map into host memory (Powers.prefix(copy=True)).  The file was just written, so its pages are in the page cache: this is
a copy from the cache, not a cold read from disk.  The setup is then timed on those copies.  Every time is the best of
--reps calls.  With --profile the largest size is run once more under torch.profiler and its kernel time is split into the
point transforms, the column sums and the rest.  The card name and power limit are read in the same command.

    python tools/bench_setup_ptau.py [--sizes 14,16,18,20] [--circuits chain,circomlike] [--reps 3] [--profile]
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
from circom_compat_b200 import CircomReduction, Context, Groth16, Powers, read_ptau, synth  # noqa: E402
from circom_compat_b200.zkey import R_MOD  # noqa: E402
import ptau_model  # noqa: E402

ARRAYS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
          'b_g2_query', 'l_query', 'h_query')


def ceremony(ctx, power, tau, alpha, beta):
    n = 1 << power
    t = [1] * (2 * n - 1)
    for i in range(1, 2 * n - 1):
        t[i] = t[i - 1] * tau % R_MOD
    fb1 = lambda v: ctx.fixed_base_g1(synth._ints_to_limbs([x % R_MOD for x in v]))  # noqa: E731
    fb2 = lambda v: ctx.fixed_base_g2(synth._ints_to_limbs([x % R_MOD for x in v]))  # noqa: E731
    return Powers(power, power, fb1(t), fb2(t[:n]), fb1([alpha * x for x in t[:n]]), fb1([beta * x for x in t[:n]]), fb2([beta]))


def best(reps, fn):
    out, t = None, None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t0
        t = dt if t is None else min(t, dt)
    return out, t


def profile(ctx, circ, pw):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        Groth16.generate_parameters_from_powers_of_tau(circ, pw, ctx)
        torch.cuda.synchronize()
    split = {'point_transforms_ms': 0.0, 'column_sums_ms': 0.0, 'other_ms': 0.0}
    for e in p.key_averages():
        us = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0)
        name = e.key
        key = 'point_transforms_ms' if 'pts_intt' in name or 'hq_circom' in name else \
              'column_sums_ms' if 'colsum' in name or 'RadixSort' in name or 'colptr' in name else 'other_ms'
        split[key] += us / 1000.0
    return {k: round(v, 2) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='14,16,18,20')
    ap.add_argument('--circuits', default='chain,circomlike')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--profile', action='store_true')
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(',')]
    print(json.dumps({'gpu': gpu_label()}), flush=True)
    ctx = Context(0)
    rng = random.Random(0x9741)
    tau, alpha, beta = (rng.randrange(1, R_MOD) for _ in range(3))
    cer = ceremony(ctx, max(sizes), tau, alpha, beta)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, 'pot.ptau')
        with open(path, 'wb') as f:
            f.write(ptau_model.write_ptau(cer.power, cer.tau_g1, cer.tau_g2, cer.alpha_tau_g1, cer.beta_tau_g1, cer.beta_g2))
        for k in sizes:
            for kind in args.circuits.split(','):
                circ = synth.chain_circuit(1 << k) if kind == 'chain' else synth.circomlike_circuit(k)[0]
                pw, t_read = best(args.reps, lambda: read_ptau(path).prefix(k, copy=True))
                pk, t_setup = best(args.reps, lambda: Groth16.generate_parameters_from_powers_of_tau(circ, pw, ctx, CircomReduction))
                ref, t_ref = best(args.reps, lambda: Groth16.generate_parameters_with_qap(circ, alpha, beta, 1, 1, tau=tau, ctx=ctx))
                if not all(np.ascontiguousarray(getattr(pk, n)).tobytes() == np.ascontiguousarray(getattr(ref, n)).tobytes()
                           for n in ARRAYS):
                    raise SystemExit(f'keys differ: {kind} 2^{k}')
                pk1, t_upd = best(args.reps, lambda: Groth16.contribute(pk, ctx=ctx))
                ok, t_chk = best(args.reps, lambda: Groth16.verify_contribution(pk, pk1, ctx))
                if not ok:
                    raise SystemExit(f'honest contribution refused: {kind} 2^{k}')
                print(json.dumps({'circuit': kind, 'log_n': k, 'n_vars': circ.n_vars, 'ptau_read_s': round(t_read, 4),
                                  'setup_from_powers_s': round(t_setup, 4), 'b2g_setup_s': round(t_ref, 4),
                                  'delta_update_s': round(t_upd, 4), 'update_check_s': round(t_chk, 4), 'identical': True}),
                      flush=True)
                del pw, pk, ref, pk1
        if args.profile:
            k = max(sizes)
            circ = synth.chain_circuit(1 << k)
            print(json.dumps({'profile': f'chain 2^{k}', **profile(ctx, circ, read_ptau(path).prefix(k, copy=True))}), flush=True)
    ctx.close()


if __name__ == '__main__':
    main()
