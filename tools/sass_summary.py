#!/usr/bin/env python
"""SASS evidence for the kernels of libkvb.so: per kernel, the counts of the mnemonics that prove what it is (bulk-copy /
mbarrier for the TMA mover, 128-bit non-allocating loads for the LDG mover, vote / popc / redux for the hash chain,
match / atomics for the index), followed by the full listing of the default gather kernel.
    python tools/sass_summary.py > sass_kernels.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "llm-d-kv-cache_b200", "libkvb.so")
WATCH = ["UBLKCP", "SYNCS", "UTMALDG", "UTMASTG", "LDG.E.128", "LDG.E.NA.128", "STG.E.128", "LDGSTS", "LDGDEPBAR", "VOTE", "POPC", "REDUX",
         "MATCH", "ATOMG", "ATOM", "RED", "BAR.SYNC", "MEMBAR", "IMAD.WIDE", "LDS", "STS", "HMMA", "UTCMMA"]


def main():
    txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    kernels = collections.OrderedDict()
    cur = None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
            continue
        if cur and re.search(r"/\*[0-9a-f]{4}\*/", line):
            kernels[cur].append(line)
    demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip() or n
    print("SASS mnemonic counts per kernel of llm-d-kv-cache_b200/libkvb.so (sm_90a), cuobjdump -sass\n")
    for name, lines in kernels.items():
        counts = collections.Counter()
        for ln in lines:
            body = ln.split("*/", 1)[1] if "*/" in ln else ln
            for w in WATCH:
                if re.search(r"\b" + re.escape(w) + r"\b", body) or (w.count(".") and w in body):
                    counts[w] += 1
        shown = ", ".join(f"{k} x{v}" for k, v in counts.items() if v)
        print(f"{demangle(name)}\n    {len(lines)} instructions; {shown}\n")
    want = "_ZN3kvb22paged_copy_bulk_kernelILi0ELi6ELi3EEEvNS_8CopyArgsE"
    print("=" * 120)
    print("full listing:", demangle(want), "(the default gather mover: mode 0 = gather, 6 stages, 3 loads in flight)")
    print("No UTMALDG / UTMASTG: the fragments are CONTIGUOUS byte runs, so the copies are 1-D bulk copies (UBLKCP, cp.async.bulk)\n"
          "completed through an mbarrier (SYNCS.ARRIVE.TRANS64 / SYNCS.PHASECHK); a tensor map would add descriptor fetches for a\n"
          "shape that has no second dimension to tile.\n")
    for ln in kernels.get(want, []):
        print(ln.rstrip())


if __name__ == "__main__":
    main()
