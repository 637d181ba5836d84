#!/bin/bash
# SASS evidence of the built extension (needs no GPU): per engine-kernel variant the Hopper / async mnemonics
SO=deepreduce_b200/ops/_dr_cuda.so
cuobjdump -sass $SO > /tmp/_dr_cuda.sass
python - <<'PY'
import re, collections
txt = open('/tmp/_dr_cuda.sass').read()
funcs = re.split(r'\n\s*Function : ', txt)[1:]
want = ['UBLKCP', 'SYNCS.ARRIVE.TRANS64', 'SYNCS.PHASECHK.TRANS64.TRYWAIT', 'SYNCS.EXCH', 'LDGSTS', 'LDGDEPBAR', 'ATOMS.POPC.INC', 'ATOMS', 'ATOMG', 'RED.E', 'REDG',
        'STG.E.128', 'STG.E.64', 'LDG.E.STRONG.SYS', 'ST.E.STRONG.SYS', 'STG.E.STRONG.SYS', 'MEMBAR.SC.SYS', 'MEMBAR.ALL.SYS', 'MEMBAR.SC.GPU', 'FENCE.VIEW.ASYNC', 'VOTE', 'POPC', 'STL', 'LDL', 'UTC', 'HMMA']
for f in funcs:
    name = f.split('\n', 1)[0].strip()
    if 'dr_engine_kernel' not in name and 'dexp_fit' not in name and 'u8_to_nhwc' not in name:
        continue
    short = re.sub(r'_ZN2dr\d+_GLOBAL__N__[0-9a-f_]+engine_cu_[0-9a-f]+', 'dr::', name)
    ops = collections.Counter()
    n = 0
    for line in f.split('\n'):
        m = re.match(r'\s+/\*[0-9a-f]+\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)', line)
        if m:
            n += 1
            op = m.group(2)
            for w in want:
                if op.startswith(w):
                    ops[w] += 1
    print(f"== {short}  ({n} SASS instructions)")
    print('   ' + ', '.join(f'{k} x{v}' for k, v in ops.items()))
PY
