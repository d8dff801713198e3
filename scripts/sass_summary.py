"""Per-kernel SASS evidence for the Hopper-native paths: counts of the wgmma (HGMMA), TMA
(UTMALDG / UTMASTG / UBLKCP) and mbarrier (SYNCS) instructions, legacy tensor instructions (HMMA)
and the MUFU / memory instructions in every kernel of libautoml_b200.so.
usage: python scripts/sass_summary.py > sass_summary.md   (no GPU needed)"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'automl_b200', 'csrc', 'libautoml_b200.so')
COLS = ['HGMMA', 'UTMALDG', 'UTMASTG', 'SYNCS', 'HMMA', 'MUFU', 'LDG', 'LDS', 'total']


def main():
  sass = subprocess.run(['cuobjdump', '-sass', LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
  kernels = collections.OrderedDict()
  cur = None
  for line in sass.splitlines():
    m = re.match(r'\s*Function : (\S+)', line)
    if m:
      cur = kernels.setdefault(m.group(1), collections.Counter())
      continue
    m = re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)', line)
    if cur is not None and m:
      op = m.group(1).split('.')[0]
      cur['total'] += 1
      if op in ('HGMMA', 'UTMALDG', 'UTMASTG', 'UBLKCP', 'SYNCS', 'HMMA', 'MUFU', 'LDG', 'LDS'):
        cur[op] += 1
  names = subprocess.run(['c++filt'], input='\n'.join(kernels), stdout=subprocess.PIPE, text=True).stdout.splitlines()
  arch = re.findall(r'arch = (sm_\w+)', sass)
  print('# SASS instruction counts per kernel (`cuobjdump -sass libautoml_b200.so`, %s only)\n' % ', '.join(sorted(set(arch))))
  print('`HGMMA` = wgmma.mma_async, `UTMALDG` / `UTMASTG` = TMA tensor load / store, '
        '`SYNCS` = mbarrier ops, `HMMA` = legacy mma.sync (none expected).\n')
  print('| kernel | ' + ' | '.join(COLS) + ' |')
  print('|---|' + '---:|' * len(COLS))
  fam = collections.OrderedDict()
  for mangled, nm in zip(kernels, names):
    short = re.sub(r'\(.*', '', nm)
    short = re.sub(r'\bvoid |edet::', '', short)
    key = re.sub(r'<.*', '', short)
    agg = fam.setdefault(key, {'n': 0, 'c': collections.Counter(), 'tmpl': []})
    agg['n'] += 1
    agg['tmpl'].append(short)
    for k, v in kernels[mangled].items():
      agg['c'][k] = max(agg['c'][k], v)
  for key, agg in fam.items():
    print('| `%s` (%d instantiations, max per instantiation) | ' % (key, agg['n']) +
          ' | '.join(str(agg['c'].get(c, 0)) for c in COLS) + ' |')
  tot = collections.Counter()
  for c in kernels.values():
    tot.update(c)
  print('\nLibrary totals: ' + ', '.join('%s %d' % (c, tot.get(c, 0)) for c in COLS))


if __name__ == '__main__':
  sys.exit(main())
