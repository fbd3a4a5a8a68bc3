#!/usr/bin/env python
"""Join an ncu SASS source page with nvdisasm line info: per CUDA source line, instructions executed
and warp-stall samples.  Usage: tools/ncu_lines.py report.ncu-rep <mangled-kernel-substring> [top]"""
import csv
import re
import subprocess
import sys
import tempfile
from collections import defaultdict
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
rep, ksub = sys.argv[1], sys.argv[2]
top = int(sys.argv[3]) if len(sys.argv) > 3 else 30

tmp = Path(tempfile.mkdtemp())
subprocess.run(["cuobjdump", "-xelf", "all", str(ROOT / "rmqtt_b200" / "libgpumqtt.so")], cwd=tmp, check=True, stdout=subprocess.DEVNULL)
dis = subprocess.run(["nvdisasm", "-g", "-c", str(tmp / "engine.sm_90a.cubin")], capture_output=True, text=True).stdout
addr2line, cur, infn = {}, None, False
SRC = {}
for ln in dis.splitlines():
    m = re.match(r"^\.text\.(\S+):", ln)
    if m:
        infn = ksub in m.group(1)
        continue
    if not infn:
        continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
    if m:
        cur = (Path(m.group(1)).name, int(m.group(2)))
        continue
    m = re.search(r"/\*([0-9a-f]{4,})\*/\s+\S", ln)
    if m and cur is not None:
        addr2line[int(m.group(1), 16)] = cur

out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr = rows[1]
ai, ii, si = hdr.index("Address"), hdr.index("Instructions Executed"), hdr.index("# Samples")
lsb = hdr.index("stall_long_sb")
base = None
per = defaultdict(lambda: [0, 0, 0])
for r in rows[2:]:
    try:
        a = int(r[ai], 16)
    except Exception:
        continue
    if base is None:
        base = a
    line = addr2line.get(a - base, ("?", 0))
    per[line][0] += int(r[ii] or 0)
    per[line][1] += int(r[si] or 0)
    per[line][2] += int(r[lsb] or 0)
def text_of(key):
    name, ln = key
    if name not in SRC:
        cand = list((ROOT / "rmqtt_b200" / "csrc").glob(name))
        SRC[name] = cand[0].read_text().splitlines() if cand else None
    src = SRC[name]
    return src[ln - 1].strip()[:100] if src and 0 < ln <= len(src) else ""
ti, ts = sum(v[0] for v in per.values()), sum(v[1] for v in per.values())
print(f"total warp-instructions {ti}, stall samples {ts}")
print("  inst%  smp%  long_sb%  line  source")
for line, v in sorted(per.items(), key=lambda kv: -(kv[1][0] / max(ti, 1) + kv[1][1] / max(ts, 1)))[:top]:
    print(f"{100 * v[0] / ti:6.1f} {100 * v[1] / ts:6.1f} {100 * v[2] / max(ts, 1):6.1f}  {line[0]}:{line[1]:<5d} {text_of(line)}")
