#!/usr/bin/env python
"""Summarise `-Xptxas -v` logs under tf_geometric_b200/csrc/build: registers / spills per kernel."""
import re, subprocess, sys, glob, os
root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tf_geometric_b200", "csrc", "build")
pat = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores.*\n.*Used (\d+) registers")
flt = sys.argv[1] if len(sys.argv) > 1 else None
for f in sorted(glob.glob(os.path.join(root, "*.ptxas.log"))):
    items = pat.findall(open(f).read())
    if not items:
        continue
    print(os.path.basename(f), "kernels:", len(items), "max regs:", max(int(i[3]) for i in items),
          "with spills:", sum(1 for i in items if int(i[2]) > 0))
    names = subprocess.run(["c++filt"], input="\n".join(i[0] for i in items), capture_output=True, text=True).stdout.split("\n")
    for (n, stack, spill, regs), d in zip(items, names):
        if (flt and flt in d) or int(spill) > 0:
            print("   regs=%s stack=%s spill=%s  %s" % (regs, stack, spill, d[:120]))
