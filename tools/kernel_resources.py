"""tools/kernel_resources.py -- `cuobjdump -res-usage` of the shipped libvb200.so, demangled,
one line per kernel instantiation (registers, per-thread stack, static shared memory, local-memory spills)."""
import re
import subprocess
import sys

so = sys.argv[1] if len(sys.argv) > 1 else "libvips_b200/libvb200.so"
txt = subprocess.run(["cuobjdump", "-res-usage", so], capture_output=True, text=True).stdout
rows = []
for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", txt):
    rows.append((m.group(1),) + tuple(int(m.group(i)) for i in range(2, 6)))
names = subprocess.run(["c++filt"], input="\n".join(r[0] for r in rows), capture_output=True, text=True).stdout.splitlines()
out = []
for name, r in zip(names, rows):
    name = re.sub(r"vb200::\(anonymous namespace\)::|vb200::|\(anonymous namespace\)::", "", name)
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)
    out.append("%-100s REG %3d  STACK %5d  SHARED %6d  LOCAL %d" % (name, r[1], r[2], r[3], r[4]))
print("# cuobjdump -res-usage %s (sm_90a), demangled, one line per kernel instantiation (tools/kernel_resources.py)." % so)
print("# LOCAL 0 everywhere: no register spills; STACK > 0 is a per-thread array the kernel declares (the 8x8 DCT workspaces, the ICC")
print("# evaluator's stage buffer) or the frame of a called slow path (double division), not a spill.")
print("\n".join(sorted(set(out))))
