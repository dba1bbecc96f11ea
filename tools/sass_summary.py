#!/usr/bin/env python
"""Per-kernel SASS summary of libliliom_b200.so (cuobjdump -sass; no GPU needed): instruction count and the mnemonics that
matter for this library — global/shared/local memory ops, barriers, atomics, fp64, and the Hopper asynchronous-copy
instructions (UBLKCP = cp.async.bulk, SYNCS = mbarrier).  usage: sass_summary.py [lib.so]"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "liliom_b200", "libliliom_b200.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
KEYS = ["LDG", "STG", "LDS", "STS", "LDL", "STL", "LDC", "BAR", "RED", "ATOM", "MEMBAR", "CCTL", "SHFL", "DFMA", "DADD", "DMUL", "FFMA", "FADD", "FMUL",
        "ISETP", "SEL", "UBLKCP", "SYNCS", "UTMALDG", "ELECT"]
cur, stats = None, collections.OrderedDict()
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1); stats[cur] = collections.Counter(); continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
    if m and cur:
        op = m.group(1)
        stats[cur]["_n"] += 1
        for k in KEYS:
            if op == k or op.startswith(k + "."):
                stats[cur][k] += 1
print(f"# {os.path.basename(lib)}: {len(stats)} kernels; columns: SASS instructions | selected mnemonic counts (zero counts omitted)")
for fn, c in stats.items():
    name = subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip() or fn
    name = re.sub(r"\(.*", "", name)[:70]
    print(f"{name:70s} {c['_n']:6d} | " + " ".join(f"{k}:{c[k]}" for k in KEYS if c[k]))
