#!/usr/bin/env python
"""Per-kernel counts of the SASS mnemonics that prove which hardware paths a kernel uses (no GPU needed: cuobjdump
reads the in-tree .so).  wgmma -> HGMMA, TMA -> UTMALDG (.2D / .4D / .MULTICAST), mbarrier -> SYNCS,
multimem.ld_reduce -> LDGMC, .sys-scope acquire/release traffic -> LDG/STG ... STRONG.SYS.

    python scripts/sass_evidence.py          (the counts go to stdout)
"""
import collections
import glob
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = sorted(glob.glob(os.path.join(ROOT, "colearn_federated_learning_b200", "ops", "_colearn_C*.so")))[0]
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
demangle = subprocess.run(["c++filt"], input="\n".join(re.findall(r"Function : (\S+)", out)), capture_output=True, text=True).stdout.splitlines()
names = iter(demangle)
pat = re.compile(r"\b(HGMMA[.\w]*|UTMALDG[.\w]*|SYNCS[.\w]*|LDGMC[.\w]*|UCGABAR\w*|"
                 r"(?:LDG|STG|ATOMG|RED)\.[.\w]*STRONG\.SYS[.\w]*|MULTIMEM[.\w]*)")
cur, counts = None, collections.OrderedDict()
for line in out.splitlines():
    if "Function :" in line:
        cur = next(names)
        cur = re.sub(r"\(anonymous namespace\)::", "", cur)
        cur = re.sub(r"\(CUtensorMap_st.*", "", cur)            # drop the parameter list
        counts[cur] = collections.Counter()
        continue
    m = pat.search(line)
    if m and cur is not None:
        counts[cur][m.group(1)] += 1
print(f"# {os.path.basename(so)} — mnemonic counts per kernel (scripts/sass_evidence.py)")
for k, c in counts.items():
    if not c:
        continue
    print(f"== {k}")
    for mn, n in c.most_common():
        print(f"{n:7d} {mn}")
