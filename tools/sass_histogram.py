"""Per-kernel SASS opcode histogram of the shipped library:
   mkdir -p profiles && python tools/sass_histogram.py > profiles/sass_opcodes.txt"""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fuzzysearch_b200", "libfuzzb200.so")
NOTABLE = re.compile(r"^(UTMA|SYNCS|ATOM|RED|MATCH|BREV|POPC|SHFL|VOTE|R2UR|LDG\.E\.128|LDS\.128|LDSM|UBLKCP|STG\.E\.128)")

out = subprocess.check_output(["cuobjdump", "-sass", LIB]).decode()
demangle = lambda s: subprocess.check_output(["c++filt", s]).decode().strip()  # noqa: E731
kernels, cur = collections.OrderedDict(), None
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = kernels.setdefault(demangle(m.group(1)), collections.Counter())
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur is not None:
        cur[m.group(1)] += 1
print("SASS opcode histogram of fuzzysearch_b200/libfuzzb200.so (cuobjdump -sass, sm_90a), per kernel.")
print("UTMALDG / SYNCS.ARRIVE.TRANS64 = TMA (cp.async.bulk.tensor) + mbarrier; LDG.E.128 = coalesced uint4 streaming loads.")
print()
for name, ops in kernels.items():
    fam = collections.Counter()
    for op, c in ops.items():
        fam[op.split(".")[0]] += c
    notable = sorted((op, c) for op, c in ops.items() if NOTABLE.match(op))
    print(name[:160])
    print("  instructions %d; top families: %s" % (sum(ops.values()), ", ".join("%s %d" % x for x in fam.most_common(12))))
    print("  notable: %s" % ", ".join("%s %d" % x for x in notable))
    print()
