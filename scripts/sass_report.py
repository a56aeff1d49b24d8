""".text bytes, registers and TMA-class instructions (UBLKCP bulk copy, UBLKPF bulk prefetch, SYNCS mbarrier) of every
kernel in the shipped library.   usage: python scripts/sass_report.py"""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ggrmcp_b200", "libggrmcp_b200.so")
elf = subprocess.run(["cuobjdump", "-elf", LIB], capture_output=True, text=True).stdout
sizes = {}
for ln in elf.splitlines():
    m = re.search(r"^\s*\w+\s+\w+\s+(\w+)\s+\w+\s+\w+\s+PROGBITS\s+\w+\s+\w+\s+\w+\s+\.text\.(\S+)", ln)
    if m:
        sizes[m.group(2)] = int(m.group(1), 16)
sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
cur = None
ops = collections.defaultdict(collections.Counter)
for ln in sass.splitlines():
    m = re.search(r"Function : (\S+)", ln)
    if m:
        cur = m.group(1)
        continue
    if cur:
        for op in ("UBLKCP", "UBLKPF", "SYNCS", "UTMALDG", "UTMASTG", "MATCH", "LDGSTS"):
            if re.search(r"\b%s\b" % op, ln) or (" " + op + ".") in ln:
                ops[cur][op] += 1
res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
regs = {}
fn = None
for ln in res.splitlines():
    m = re.search(r"Function (\S+):", ln)
    if m:
        fn = m.group(1)
    m = re.search(r"REG:(\d+).*?SHARED:(\d+)", ln)
    if m and fn:
        regs[fn] = (int(m.group(1)), int(m.group(2)))
dem = subprocess.run(["c++filt"] + list(sizes), capture_output=True, text=True).stdout.splitlines()
names = dict(zip(sizes, dem))
print("# kernels of ggrmcp_b200/libggrmcp_b200.so (sm_90a): .text bytes, registers, static shared memory, bulk / TMA-class SASS")
print("%-9s %5s %7s  %-22s %s" % (".text", "regs", "smem", "UBLKCP/UBLKPF/SYNCS", "kernel"))
for k, v in sorted(sizes.items(), key=lambda kv: -kv[1]):
    r = regs.get(k, (0, 0))
    o = ops.get(k, {})
    short = re.sub(r"\(.*", "", names.get(k, k))
    print("%-9d %5d %7d  %-22s %s" % (v, r[0], r[1], "%d/%d/%d" % (o.get("UBLKCP", 0), o.get("UBLKPF", 0), o.get("SYNCS", 0)), short))
