"""Witnesses/s of WitnessCalculator.calculate_witnesses (circom 2 .wasm run by the device interpreter, one lane per
witness) for the reference's two circom 2 fixtures, mycircuit and circuit2, at several counts, and the latency of a
single witness.  For scale it also times the plain-Python model (tests/wasm_model.py) on one host core.

Every count is warmed up once, then timed --rounds times with a host clock around the synchronous call (inputs packed
and hashed on the host, the upload, the kernels and the download included); the best round is the figure.  Each cell
checks a sample of its witnesses (w[1] = a * b).  One JSON line per cell goes to stdout and, with --out, to that file;
the first line records the card and its power limit.  The last line times one lane spinning in a loop until its fuel runs
out, which is how long the default fuel cap lets a runaway lane hold a call.

    python tools/bench_witness.py [--counts 1,1024,16384,65536] [--rounds 3] [--model-witnesses 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(',')]
    return {'gpu': name, 'power_limit': power, 'max_sm_clock': clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,1024,16384,65536')
    ap.add_argument('--circuits', default='mycircuit,circuit2')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--model-witnesses', type=int, default=3)
    ap.add_argument('--out')
    a = ap.parse_args()
    from circom_compat_b200 import Context, WitnessCalculator, fr_from_mont
    from circom_compat_b200.zkey import R_MOD
    import wasm_model
    out = open(a.out, 'w') if a.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + '\n')
            out.flush()
    emit({'card': card()})
    ctx = Context(0)
    rng = random.Random(1)
    for name in a.circuits.split(','):
        data = open(os.path.join(GOLDEN, name + '.wasm'), 'rb').read()
        calc = WitnessCalculator.new(data, ctx)
        for count in [int(x) for x in a.counts.split(',')]:
            ins = [{'a': rng.randrange(2, 1 << 64), 'b': rng.randrange(2, 1 << 64)} for _ in range(count)]
            calc.calculate_witnesses(ins[:min(count, 32)])               # warm-up (module load, first launch)
            best = None
            for _ in range(a.rounds):
                t = time.perf_counter()
                wm, st = calc.calculate_witnesses(ins)
                dt = time.perf_counter() - t
                best = dt if best is None else min(best, dt)
            assert not st.any(), f"{name}: {int((st != 0).sum())} lanes failed"
            for i in {0, count - 1, count // 2}:
                w = fr_from_mont(wm[i][:16])
                assert w[1] == ins[i]['a'] * ins[i]['b'] % R_MOD and w[2] == ins[i]['a']
            emit({'circuit': name, 'count': count, 'best_s': round(best, 6), 'witnesses_per_s': round(count / best, 1),
                  'witness_size': calc.witness_size, 'rounds': a.rounds})
        calc.close()
        if a.model_witnesses:
            model = wasm_model.Calculator(data)
            t = time.perf_counter()
            for k in range(a.model_witnesses):
                st, _ = model.calculate([('a', [3 + k]), ('b', [11])])
                assert st == 0
            dt = time.perf_counter() - t
            emit({'circuit': name, 'python_model_one_core_witnesses_per_s': round(a.model_witnesses / dt, 2)})
    # how long the fuel cap lets a runaway lane run: one lane in a one-instruction loop until its fuel is spent
    import wasm_asm as A
    from circom_compat_b200 import WasmModule
    spin = WasmModule(A.module([A.Func([], [], b'\x03\x40\x0c\x00\x0b', export='spin')]), ctx)
    spin.set_limits(fuel=1 << 16)
    spin.run('spin', [()])                                                # warm-up
    fuel = 1 << 26
    spin.set_limits(fuel=fuel)
    t = time.perf_counter()
    _, st = spin.run('spin', [()])
    dt = time.perf_counter() - t
    assert st[0] == wasm_model.FUEL
    emit({'runaway_lane_fuel': fuel, 'seconds': round(dt, 3), 'instructions_per_s': round(fuel / dt, 1),
          'default_fuel_2p32_seconds': round((1 << 32) / (fuel / dt), 1)})
    spin.close()
    ctx.close()


if __name__ == '__main__':
    main()
