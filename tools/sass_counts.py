#!/usr/bin/env python3
"""SASS opcode histogram per kernel of libalgebra_b200.so (cuobjdump -sass): the evidence for "hand-written integer kernels":
IMAD.WIDE counts, LDGSTS (cp.async).  usage: sass_counts.py [kernel-name-regex]"""
import collections, os, re, subprocess, sys
so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "algebra_b200", "libalgebra_b200.so")
pat = re.compile(sys.argv[1] if len(sys.argv) > 1 else r"msm_pair_add|ntt_pass|msm_accumulate_kernel<ab200::CurveBls,|msm_digits")
sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
cur, cnt = None, collections.OrderedDict()
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        cur = name if pat.search(name) else None
        if cur:
            cnt[cur] = collections.Counter()
        continue
    m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        cnt[cur][m.group(1)] += 1
for k, c in cnt.items():
    tot = sum(c.values())
    wide = sum(v for o, v in c.items() if o.startswith("IMAD.WIDE"))
    key = {o: v for o, v in c.items() if o.startswith(("IMAD", "LDGSTS", "LDG", "STG", "LDS", "STS", "BAR", "SHFL", "CALL"))}
    print(f"{k[:140]}\n  total {tot}  IMAD.WIDE* {wide} ({100.0 * wide / tot:.1f} %)  " + "  ".join(f"{o}:{v}" for o, v in sorted(key.items(), key=lambda kv: -kv[1])[:14]))
