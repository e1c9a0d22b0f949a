"""Preparing many verifying keys: a loop of b2g_vk_load (one key per call) against one b2g_vk_load_many call, and a first
b2g_verify_batch_keys call over K fresh keys x 1 proof with its keys loaded one by one (the route the keyed verifiers took
before b2g_vk_load_many) against loaded in one call.

Keys and proofs are made with known discrete logs on the device (Context.fixed_base_g1 / g2, as in bench_verify_keys.py); the
descriptors, public inputs, proofs and weights are encoded once, and every arm goes through the C ABI.  Every handle is freed
between repetitions (untimed), so each repetition loads fresh keys.  A time is the best of --reps calls; the arms that loop
over 1 024 or more keys run once (each such run takes seconds).  --parent-lib adds the loop arms once more through another
build of the library (e.g. the commit before b2g_vk_load_many), with a context of its own.

    python tools/bench_vk_load.py [--reps 3] [--parent-lib PATH]
"""
import argparse
import ctypes as C
import json
import os
import secrets
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_verify import gpu_label  # noqa: E402
from bench_verify_keys import make_keys  # noqa: E402
from circom_compat_b200 import Context  # noqa: E402
from circom_compat_b200 import _native as N  # noqa: E402
from circom_compat_b200.groth16 import _vk_desc  # noqa: E402

LOAD_SIZES = [(1, k) for k in (1, 16, 256, 1024, 4096)] + [(100, k) for k in (1, 16, 64)]
VERIFY_SIZES = (1, 16, 256, 1024)
LONG = 1024                                             # loop arms over this many keys or more run once


class Lib:
    """the entry points the loop arms need, from a build of the library given by path, with a context of its own"""

    def __init__(self, path):
        L = C.CDLL(path)
        vp = C.c_void_p
        L.b2g_last_error.restype = C.c_char_p
        L.b2g_ctx_create.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
        L.b2g_ctx_destroy.argtypes = [vp]
        L.b2g_vk_load.argtypes = [vp, C.POINTER(N.VkDesc), C.POINTER(vp)]
        L.b2g_vk_free.argtypes = [vp]
        L.b2g_verify_batch_keys.argtypes = [vp, C.c_uint32, C.POINTER(N.KeyBatch), vp]
        self.L, self.ctx = L, vp()
        self.check(L.b2g_ctx_create(0, 0, 1, C.byref(self.ctx)))

    def check(self, rc):
        if rc:
            raise N.B2gError(rc, self.L.b2g_last_error().decode())


def _ptr(a):
    return a.ctypes.data if a is not None and a.size else None


def _arr(b):
    return np.frombuffer(b, dtype=np.uint8).copy() if b else None


def load_loop(lib, ctx, descs):
    hs = []
    for d in descs:
        h = C.c_void_p()
        lib.check(lib.L.b2g_vk_load(ctx, C.byref(d), C.byref(h)))
        hs.append(h)
    return hs


def load_many(ctx, descs):
    out = (C.c_void_p * len(descs))()
    N.check(N.lib().b2g_vk_load_many(ctx._h, len(descs), descs, out))
    return [C.c_void_p(h) for h in out]


def free(lib, hs):
    for h in hs:
        lib.L.b2g_vk_free(h)


def verify_first(lib, ctx, load, descs, batches):
    """load the keys, then one b2g_verify_batch_keys over one proof per key; all verdicts must be 1.  Returns the handles."""
    hs = load()
    table = (N.KeyBatch * len(hs))(*[N.KeyBatch(h.value, 1, 0, _ptr(pub), _ptr(pr), _ptr(w)) for h, (pub, pr, w) in zip(hs, batches)])
    verdicts = np.zeros(len(hs), dtype=np.uint8)
    lib.check(lib.L.b2g_verify_batch_keys(ctx, len(hs), table, verdicts.ctypes.data))
    assert verdicts.all()
    return hs


def best_ms(fn, lib, reps):
    """the best of reps timed runs of fn (which returns handles; they are freed after each run, untimed)"""
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        hs = fn()
        dt = time.perf_counter() - t0
        free(lib, hs)
        best = dt if best is None else min(best, dt)
    return round(best * 1e3, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--parent-lib', default=None)
    args = ap.parse_args()
    ctx = Context(0)
    this = Lib(N.LIB_PATH)
    parent = Lib(args.parent_lib) if args.parent_lib else None
    print(f'# GPU: {gpu_label()}', flush=True)
    libs = [('loop', this, this.ctx)] + ([('parent_loop', parent, parent.ctx)] if parent else [])
    for n_public in (1, 100):
        n_max = max(k for p, k in LOAD_SIZES if p == n_public)
        keys = make_keys(ctx, n_max, n_public, 1, 11 + n_public)
        pairs = [_vk_desc(vk) for vk, _, _ in keys]
        all_descs = (N.VkDesc * n_max)(*[d for d, _ in pairs])
        batches = [(_arr(pubs[0]), _arr(proofs[0]), _arr((secrets.randbits(128) | 1).to_bytes(16, 'little'))) for _, pubs, proofs in keys]
        one = (N.VkDesc * 1)(all_descs[0])
        for _, lib, lctx in libs:                                # warm-up: module loads and the first allocations
            free(lib, load_loop(lib, lctx, one))
        free(this, load_many(ctx, one))
        for p, k in LOAD_SIZES:
            if p != n_public:
                continue
            descs = (N.VkDesc * k)(*all_descs[:k])
            reps = 1 if k >= LONG else args.reps
            row = {'n_public': n_public, 'keys': k}
            for label, lib, lctx in libs:
                row[f'{label}_ms'] = best_ms(lambda: load_loop(lib, lctx, descs), lib, reps)
            row['many_ms'] = best_ms(lambda: load_many(ctx, descs), this, args.reps)
            row['many_speedup_over_loop'] = round(row['loop_ms'] / row['many_ms'], 1)
            if n_public == 1 and k in VERIFY_SIZES:
                for label, lib, lctx in libs:
                    row[f'first_verify_{label}_ms'] = best_ms(
                        lambda: verify_first(lib, lctx, lambda: load_loop(lib, lctx, descs), descs, batches[:k]), lib, reps)
                row['first_verify_many_ms'] = best_ms(
                    lambda: verify_first(this, this.ctx, lambda: load_many(ctx, descs), descs, batches[:k]), this, args.reps)
                hs = load_many(ctx, descs)
                row['verify_only_ms'] = best_ms(lambda: verify_first(this, this.ctx, lambda: hs, descs, batches[:k]) and [], this, args.reps)
                free(this, hs)
            print(json.dumps(row), flush=True)
    for lib in (this, parent):
        if lib:
            lib.L.b2g_ctx_destroy(lib.ctx)
    ctx.close()


if __name__ == '__main__':
    main()
