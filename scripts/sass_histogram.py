#!/usr/bin/env python
"""SASS opcode histogram of libkge_b200.so, per kernel (static instruction counts), and the Hopper-specific
mnemonics that prove which engines a kernel uses (UBLKCP = cp.async.bulk, HGMMA = wgmma, REDG = red.global,
SYNCS = mbarrier, LDGMC = multimem.ld_reduce).  Usage: python scripts/sass_histogram.py [so] > ncu_out/<tag>_sass_opcodes.txt"""
import collections
import re
import subprocess
import sys

so = sys.argv[1] if len(sys.argv) > 1 else "ampligraph_b200/libkge_b200.so"
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
kern, hist = None, collections.OrderedDict()
for line in txt.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        kern = re.sub(r"\(.*", "", name).replace("void ", "").replace("kge::", "")
        hist[kern] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
    if m and kern:
        hist[kern][m.group(1)] += 1
MARK = ("UBLKCP", "UBLKRED", "HGMMA", "WARPGROUP", "UTMALDG", "REDG", "SYNCS", "HMMA", "LDGSTS", "LDGMC")
print("# static SASS opcode counts per kernel of %s (cuobjdump -sass); marker mnemonics first, then the ten most frequent" % so)
for k, h in hist.items():
    tot = sum(h.values())
    marks = " ".join("%s=%d" % (m, sum(v for op, v in h.items() if op.startswith(m))) for m in MARK if any(op.startswith(m) for op in h))
    top = " ".join("%s=%d" % kv for kv in h.most_common(10))
    print("%-70s total=%-6d | %s | %s" % (k[:70], tot, marks, top))
