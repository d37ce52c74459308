"""Counts the SASS mnemonics that show what the kernels are made of (cuobjdump -sass of the built library).
    python scripts/sass_excerpt.py > sass_excerpt.txt"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "libdeflate_b200", "libdeflate_b200.so")
out = subprocess.run(["cuobjdump", "-sass", so], stdout=subprocess.PIPE, text=True).stdout
want = re.compile(r"^(UBLKCP|SYNCS|IDP|MATCH|REDUX|VOTE|VOTEU|SHFL|ATOM|ATOMS|ATOMG|RED|LDGSTS|LDGDEPBAR|DEPBAR|LDS\.128|STS\.128|STG\.E\.128|LDG\.E\.128|UTC|HMMA|IMMA)")
fn, per = None, collections.OrderedDict()
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        fn = m.group(1); per[fn] = collections.Counter(); continue
    m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", line)
    if m and fn and want.match(m.group(1)):
        per[fn][m.group(1)] += 1
print("# SASS mnemonics of libdeflate_b200.so (cuobjdump -sass, sm_90a), count per kernel (scripts/sass_excerpt.py)")
print("# 1-D bulk TMA (UBLKCP) + mbarrier (SYNCS) in the deflate kernel, asynchronous global->shared copies (LDGSTS + LDGDEPBAR/DEPBAR) in the")
print("# decode kernel, dp4a in Adler-32, warp votes / shuffles / match / redux throughout; no tensor-core mnemonics (UTC*MMA / HMMA):")
print("# this is integer / byte work")
for fn, c in per.items():
    print(fn)
    print("   " + ", ".join("%s x%d" % kv for kv in sorted(c.items())))
