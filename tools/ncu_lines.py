#!/usr/bin/env python
"""Attribute ncu per-SASS-instruction counts (ncu -i X.ncu-rep --page source --csv) to CUDA source lines using
nvdisasm -g line info of the same cubin.  Usage: ncu_lines.py <src.csv> <kernel substring> <sass file> [top]"""
import csv, os, re, sys
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tokenizers_b200", "csrc")
src_csv, kname, sass, top = sys.argv[1], sys.argv[2], sys.argv[3], int(sys.argv[4]) if len(sys.argv) > 4 else 40
rows = list(csv.reader(open(src_csv)))
h = rows[1]; ix = h.index("Instructions Executed"); ns = h.index("# Samples"); tx = h.index("Thread Instructions Executed")
data = [r for r in rows[2:] if len(r) > ix and r[ix].isdigit()]
# sass: find function section
lines = open(sass).read().split("\n")
infn = False; cur = None; insn_lines = []
for ln in lines:
    if re.match(r"\s*\.section\s+\.(text|nv)", ln) or ln.startswith("//-----"):
        if ".text." in ln: infn = kname in ln
        elif ln.startswith("//-----") or ".section" in ln: infn = infn and (kname in ln)
        continue
    if not infn: continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
    if m: cur = (m.group(1).split("/")[-1], int(m.group(2))); continue
    if re.match(r"\s+/\*[0-9a-f]{4,}\*/", ln): insn_lines.append(cur)
print("sass instrs", len(insn_lines), "ncu rows", len(data))
agg = {}
tot = sum(int(r[ix]) for r in data)
for r, loc in zip(data, insn_lines):
    a = agg.setdefault(loc, [0, 0, 0]); a[0] += int(r[ix]); a[1] += int(r[ns]); a[2] += int(r[tx])
srcs = {}
for (loc, a) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:top]:
    if loc is None: print("?", a); continue
    f, l = loc
    if f not in srcs:
        try: srcs[f] = open(os.path.join(CSRC, f)).read().split("\n")
        except Exception: srcs[f] = []
    text = srcs[f][l - 1].strip()[:110] if l - 1 < len(srcs[f]) else ""
    print(f"{100.0 * a[0] / tot:5.1f}% inst  {a[1]:6d} samples  lanes {a[2] / max(a[0], 1):4.1f}  {f}:{l}  {text}")
