"""Per-kernel counts of the Hopper-native SASS instructions in libvalle_b200.so (cuobjdump -sass):
HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / arrive / wait, UTMALDG/UTMASTG/UTMAREDG = TMA tensor
load/store/reduce, UBLKCP = cp.async.bulk, UTMAPF = TMA descriptor prefetch, SYNCS = mbarrier operations,
HMMA = warp-level mma.sync, LDGSTS = cp.async.

    python tools/sass_summary.py [lib.so] [--match REGEX]

--match lists the total instruction count of every kernel whose demangled name matches REGEX instead (e.g.
`--match "layernorm_kernel|ln_reduce_kernel"` to compare the instantiations of two builds).
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
args = sys.argv[1:]
match = None
if "--match" in args:
    i = args.index("--match")
    match = re.compile(args[i + 1])
    del args[i:i + 2]
lib = args[0] if args else os.path.join(ROOT, "valle_b200", "lib", "libvalle_b200.so")
PAT = re.compile(r"\b(HGMMA|WARPGROUP|UTMALDG|UTMASTG|UTMAREDG|UBLKCP|UTMAPF|SYNCS|HMMA|LDGSTS)\b")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
cur, tab = None, collections.OrderedDict()
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        tab[cur] = collections.Counter()
        continue
    if cur:
        for op in PAT.findall(line):
            tab[cur][op] += 1
        tab[cur]["_instr"] += 1 if re.search(r"/\*[0-9a-f]{4}\*/", line) else 0
dem = subprocess.run(["c++filt"], input="\n".join(tab), capture_output=True, text=True).stdout.splitlines()
if match is not None:
    print(f"# {os.path.relpath(lib, ROOT)}: SASS instructions per kernel (cuobjdump -sass, sm_90a)")
    for (name, cnt), d in sorted(zip(tab.items(), dem), key=lambda t: t[1]):
        if match.search(d):
            print(f"{cnt['_instr']:8d}  {d}")
    sys.exit(0)
cols = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAREDG", "UBLKCP", "UTMAPF", "SYNCS", "HMMA", "LDGSTS"]
print(f"# {os.path.relpath(lib, ROOT)}: SASS instruction counts per kernel (cuobjdump -sass, sm_90a)")
print(f"{'kernel':90s} " + " ".join(f"{c:>8s}" for c in cols))
tot = collections.Counter()
for (name, cnt), d in zip(tab.items(), dem):
    short = re.sub(r"\(.*", "", d)[:90]
    if not any(cnt[c] for c in cols):
        continue
    print(f"{short:90s} " + " ".join(f"{cnt[c]:8d}" for c in cols))
    tot.update({c: cnt[c] for c in cols})
print(f"{'TOTAL':90s} " + " ".join(f"{tot[c]:8d}" for c in cols))
