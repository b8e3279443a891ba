"""cuobjdump -sass of the in-tree library -> per kernel: instruction count and the mnemonics that prove the Hopper paths.
usage (no GPU needed): python tools/sass_evidence.py"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, 'renet_b200', 'librenet_b200.so')
out = subprocess.run(['cuobjdump', '-sass', so], capture_output=True, text=True).stdout
names = subprocess.run(['c++filt'], input='\n'.join(re.findall(r'Function : (\S+)', out)), capture_output=True, text=True).stdout.splitlines()
KEYS = ('HGMMA', 'WARPGROUP', 'UBLKCP', 'UTMALDG', 'SYNCS', 'LDGSTS', 'ATOMS', 'ATOMG', 'RED', 'HMMA', 'ELECT')
rows, cur, it = [], None, iter(names)
for line in out.splitlines():
    m = re.search(r'Function : (\S+)', line)
    if m:
        cur = [next(it), 0, collections.Counter()]
        rows.append(cur)
        continue
    if cur is None:
        continue
    m = re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)', line)
    if m:
        cur[1] += 1
        op = m.group(1)
        for k in KEYS:
            if op.startswith(k):
                cur[2][k if k != 'ATOMS' else '.'.join(op.split('.')[:3])] += 1
print('# cuobjdump -sass renet_b200/librenet_b200.so (sm_90a), per kernel: instruction count and the mnemonics that prove the')
print('# wgmma / TMA paths (HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / wait, UBLKCP = cp.async.bulk,')
print('# SYNCS = mbarrier ops, ELECT = elect.sync) and the absence / presence of shared-memory atomics (ATOMS.*)')
for name, n, c in sorted(rows, key=lambda r: -r[1]):
    if name.startswith('void cub::') or 'cub::' in name[:30]:
        continue
    print('%-150s %6d instr  %s' % (name[:150], n, ' '.join('%s=%d' % kv for kv in sorted(c.items()))))
