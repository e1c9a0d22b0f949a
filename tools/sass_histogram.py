#!/usr/bin/env python
"""Per-kernel SASS instruction histogram of libb2groth.so (cuobjdump -sass), the static evidence behind the pipe-bound
claims in DESIGN.md: how many IMAD.WIDE (the 32x32->64 multiply-add the fmaheavy pipe issues once per 4 cycles per SM
sub-partition), other IMAD-class instructions (same pipe, half cost), integer adds, global loads by width, and
local-memory (stack) loads / stores each kernel contains.  Usage: python tools/sass_histogram.py [lib.so]"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'circom_compat_b200', 'libb2groth.so')
sass = subprocess.check_output(['cuobjdump', '-sass', lib], text=True, errors='replace')
try:
    import cxxfilt  # noqa: F401
except Exception:
    cxxfilt = None


def demangle(names):
    try:
        out = subprocess.check_output(['c++filt'] + names, text=True).splitlines()
        return dict(zip(names, out))
    except Exception:
        return {n: n for n in names}


kernels = collections.OrderedDict()
cur = None
for line in sass.splitlines():
    m = re.match(r'\s*Function : (\S+)', line)
    if m:
        cur = m.group(1); kernels[cur] = collections.Counter(); continue
    m = re.match(r'\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)', line)
    if m and cur:
        kernels[cur][m.group(1)] += 1

names = demangle(list(kernels))
cols = ['total', 'IMAD.WIDE', 'IMAD other', 'IADD3/IADD', 'LOP3/SHF/SEL', 'LDG.128', 'LDG.256', 'LDG other', 'LDS/STS', 'LDL', 'STL', 'SHFL', 'BAR', 'CALL']
print('# cuobjdump -sass', os.path.relpath(lib, ROOT), '(sm_90a).  Static instruction counts per kernel / device function.')
print('# IMAD.WIDE = IMAD.WIDE(.U32)(.X); "IMAD other" = IMAD / IMAD.X / IMAD.MOV / IMAD.SHL / IMAD.IADD / IMAD.HI (same pipe); LDL/STL = local (stack) traffic')
print('%-74s' % 'function' + ''.join('%13s' % c for c in cols))
for k, cnt in kernels.items():
    tot = sum(cnt.values())
    wide = sum(v for o, v in cnt.items() if o.startswith('IMAD.WIDE'))
    imad = sum(v for o, v in cnt.items() if o.startswith('IMAD')) - wide
    iadd = sum(v for o, v in cnt.items() if o.startswith('IADD'))
    logic = sum(v for o, v in cnt.items() if o.split('.')[0] in ('LOP3', 'SHF', 'SEL', 'ISETP', 'PRMT', 'MOV'))
    ldg128 = sum(v for o, v in cnt.items() if o.startswith('LDG') and '.128' in o)
    ldg256 = sum(v for o, v in cnt.items() if o.startswith('LDG') and ('.256' in o or '.ENL2.256' in o))
    ldg = sum(v for o, v in cnt.items() if o.startswith('LDG')) - ldg128 - ldg256
    lds = sum(v for o, v in cnt.items() if o.startswith('LDS') or o.startswith('STS'))
    ldl = sum(v for o, v in cnt.items() if o.startswith('LDL'))
    stl = sum(v for o, v in cnt.items() if o.startswith('STL'))
    shfl = sum(v for o, v in cnt.items() if o.startswith('SHFL'))
    bar = sum(v for o, v in cnt.items() if o.startswith('BAR'))
    call = sum(v for o, v in cnt.items() if o.startswith('CALL'))
    name = names.get(k, k)
    name = re.sub(r'b2g::', '', name)
    name = re.sub(r'\(.*$', '', name)
    vals = [tot, wide, imad, iadd, logic, ldg128, ldg256, ldg, lds, ldl, stl, shfl, bar, call]
    print('%-74s' % name[:73] + ''.join('%13d' % v for v in vals))
