"""Registers / spills of every kernel in a .cu file: python scripts/ptxas_table.py body_kernels.cu [-DB200_TUNE] [filter]"""
import re, subprocess, sys, os
here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "elodin_b200", "csrc")
src = sys.argv[1]
flags = [a for a in sys.argv[2:] if a.startswith("-")]
filt = [a for a in sys.argv[2:] if not a.startswith("-")]
out = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xptxas", "-v", *flags,
                      "-c", src, "-o", "/tmp/ptxas_table.o"], cwd=here, capture_output=True, text=True).stderr
name = None
rows = []
for line in out.splitlines():
    m = re.search(r"Compiling entry function '(\S+)'", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        name = re.sub(r"\(.*", "", name).replace("void b200::", "")
        continue
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
    if m:
        spill = (int(m.group(2)), int(m.group(3)))
        continue
    m = re.search(r"Used (\d+) registers", line)
    if m and name:
        rows.append((name, int(m.group(1)), spill))
        name = None
for n, r, s in rows:
    if all(f in n for f in filt):
        print(f"{n:90s} regs {r:4d}  spill st/ld {s[0]:4d}/{s[1]:4d}")
