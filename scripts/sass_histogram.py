#!/usr/bin/env python
"""cuobjdump -sass of libshifu_b200.so -> opcode histogram per kernel family (what shows a Hopper-native kernel:
HGMMA = wgmma, UTMALDG/UTMASTG = TMA, SYNCS = mbarrier, HMMA = the older warp-level mma).

    python scripts/sass_histogram.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "shifu-tensorflow_b200", "lib", "libshifu_b200.so")
KEY = ("UTCHMMA", "UTCQMMA", "UTCBAR", "UTCCP", "LDTM", "STTM", "UTMALDG", "UTMASTG", "UTMAPF", "UBLKCP", "SYNCS", "HMMA", "HGMMA",
       "REDG", "RED.", "ATOMG", "MULTIMEM", "LDGSTS", "UCGABAR", "ACQBULK", "UTMACCTL", "ELECT", "PLOP3", "LD.E", "ST.E", "LDG", "STG")


def main():
    txt = subprocess.run(["cuobjdump", "-sass", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    fam = collections.OrderedDict()
    cur = None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], stdout=subprocess.PIPE, text=True).stdout.strip()
            name = re.sub(r"\(.*", "", name)
            cur = fam.setdefault(name, collections.Counter())
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
        if m and cur is not None:
            cur[m.group(1)] += 1
            cur["#instructions"] += 1
    print("# cuobjdump -sass %s : opcode counts per kernel (full mnemonic incl. modifiers), tensor / TMA / TMEM / atomics only" %
          os.path.relpath(LIB, ROOT))
    tot = collections.Counter()
    for name, cnt in fam.items():
        keep = {k: v for k, v in cnt.items() if any(k.startswith(p) for p in KEY)}
        if not any(k.startswith(("HGMMA", "UTMA", "MULTIMEM", "HMMA")) for k in keep) and "gemm" not in name and "xchg" not in name and "allreduce" not in name:
            continue
        print("\n%s   [%d SASS instructions]" % (name, cnt["#instructions"]))
        for k in sorted(keep):
            print("    %-44s %6d" % (k, keep[k]))
            tot[k] += keep[k]
    print("\n# totals over the listed kernels")
    for k in sorted(tot):
        print("    %-44s %6d" % (k, tot[k]))
    legacy = sum(v for k, v in tot.items() if k.startswith("HMMA"))
    print("\n# warp-level tensor path (HMMA) instructions: %d" % legacy)


if __name__ == "__main__":
    main()
