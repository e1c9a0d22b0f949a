"""Groth16 setup: one b2g_setup call (Groth16.generate_parameters_with_qap, every scalar and point on the device) against the
path it replaces, synth.setup (the scalars with big-int Python loops on one core, their packing into limbs, then the
fixed-base products on the GPU).  Both keys are compared byte for byte in the same run before anything is reported.

Circuits: synth.chain_circuit and synth.circomlike_circuit, domains 2^k for k in --sizes, under both reductions.  The
b2g_setup time is the best of --reps calls (host descriptor building included); the synth.setup time is one call.  The card
name and power limit are read in the same command.

    python tools/bench_setup.py [--sizes 14,16,18,20,22] [--reps 3] [--circuits chain,circomlike]
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

from bench_verify import gpu_label  # noqa: E402
from circom_compat_b200 import CircomReduction, Context, Groth16, LibsnarkReduction, synth  # noqa: E402
from circom_compat_b200.zkey import R_MOD  # noqa: E402

ARRAYS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
          'b_g2_query', 'l_query', 'h_query')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='14,16,18,20,22')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--circuits', default='chain,circomlike')
    args = ap.parse_args()
    print(json.dumps({'gpu': gpu_label()}), flush=True)
    ctx = Context(0)
    rng = random.Random(0x5E7)
    for k in (int(x) for x in args.sizes.split(',')):
        for kind in args.circuits.split(','):
            circ = synth.chain_circuit(1 << k) if kind == 'chain' else synth.circomlike_circuit(k)[0]
            for red, flavour in ((CircomReduction, 'circom'), (LibsnarkReduction, 'libsnark')):
                alpha, beta, gamma, delta, tau = (rng.randrange(1, R_MOD) for _ in range(5))
                best = None
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    pk = Groth16.generate_parameters_with_qap(circ, alpha, beta, gamma, delta, tau=tau, ctx=ctx, reduction=red)
                    dt = time.perf_counter() - t0
                    best = dt if best is None else min(best, dt)
                t0 = time.perf_counter()
                ref, _ = synth.setup(ctx, circ, trapdoor=(tau, alpha, beta, gamma, delta), flavour=flavour)
                old = time.perf_counter() - t0
                same = all(np.ascontiguousarray(getattr(pk, n)).tobytes() == np.ascontiguousarray(getattr(ref, n)).tobytes()
                           for n in ARRAYS)
                if not same:
                    raise SystemExit(f'keys differ: {kind} 2^{k} {flavour}')
                print(json.dumps({'circuit': kind, 'log_n': k, 'reduction': flavour, 'n_vars': circ.n_vars,
                                  'b2g_setup_s': round(best, 4), 'synth_setup_s': round(old, 3), 'speedup': round(old / best, 1),
                                  'identical': same}), flush=True)
    ctx.close()


if __name__ == '__main__':
    main()
