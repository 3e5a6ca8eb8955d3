#!/usr/bin/env python
"""Sum ncu per-SASS-instruction counts and stall samples of the page kernel by phase (source-line ranges of
model_kernels.cuh).  Usage: ncu_phases.py <src.csv> <kernel substring> <sass file>"""
import csv, os, re, sys
src_csv, kname, sass = sys.argv[1], sys.argv[2], sys.argv[3]
rows = list(csv.reader(open(src_csv)))
h = rows[1]; ix = h.index("Instructions Executed"); ns = h.index("# Samples"); tx = h.index("Thread Instructions Executed")
sb = h.index("stall_barrier"); sl = h.index("stall_long_sb")
data = [r for r in rows[2:] if len(r) > ix and r[ix].isdigit()]
lines = open(sass).read().split("\n")
infn = False; cur = None; locs = []
for ln in lines:
    if re.match(r"\s*\.section\s+\.(text|nv)", ln) or ln.startswith("//-----"):
        if ".text." in ln: infn = kname in ln
        elif ln.startswith("//-----") or ".section" in ln: infn = infn and (kname in ln)
        continue
    if not infn: continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
    if m: cur = (m.group(1).split("/")[-1], int(m.group(2))); continue
    if re.match(r"\s+/\*[0-9a-f]{4,}\*/", ln): locs.append(cur)
src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tokenizers_b200", "csrc", "model_kernels.cuh")).read().split("\n")
# phase markers: a phase starts at the first line containing the marker text
marks = [("wc_make_key", "__device__ __forceinline__ void wc_make_key"), ("wc_lookup", "__device__ __forceinline__ bool wc_lookup"),
         ("wc_publish", "__device__ __forceinline__ void wc_publish"), ("vocab_whole", "__device__ __forceinline__ bool vocab_whole_word"),
         ("coop_bpe", "__device__ __forceinline__ void coop_bpe"), ("kernel_head", "model_tile_kernel(const ModelParams P)"),
         ("P0 stage", "P0: stage bytes"), ("P1/P2 prefixes", "P1/P2: prefixes"), ("s_pt list + longs", "const int Pn = s_P;"),
         ("P3 cache lookup loop", "P3: word cache, one pre-token"), ("P4 misses", "P4a: misses"), ("P4b warp", "P4b: one warp per longer"),
         ("WordPiece", "WordPiece P3"), ("P5 token bitmap", "P5: token bitmap"), ("P6/P7 emit", "const unsigned long long excl = s_excl;"),
         ("P8 row_ptr", "P8: row_ptr"), ("pass2", "pass 2")]
starts = []
for name, text in marks:
    for i, l in enumerate(src):
        if text in l: starts.append((i + 1, name)); break
starts.sort()
def phase(loc):
    if loc is None: return "?"
    f, l = loc
    if f != "model_kernels.cuh": return f
    if l < starts[0][0]: return "merge_lookup/helpers"
    nm = None
    for s, n in starts:
        if l >= s: nm = n
    return nm
agg = {}
tot = sum(int(r[ix]) for r in data); tots = sum(int(r[ns]) for r in data)
for r, loc in zip(data, locs):
    a = agg.setdefault(phase(loc), [0, 0, 0, 0, 0]); a[0] += int(r[ix]); a[1] += int(r[ns]); a[2] += int(r[tx]); a[3] += int(r[sb] or 0); a[4] += int(r[sl] or 0)
print(f"total warp-instr {tot}, samples {tots}")
for k, a in sorted(agg.items(), key=lambda kv: -kv[1][0]):
    print(f"{100.0 * a[0] / tot:5.1f}% inst  {100.0 * a[1] / tots:5.1f}% samples  lanes {a[2] / max(a[0], 1):4.1f}  barrier {100.0 * a[3] / tots:4.1f}%  long_sb {100.0 * a[4] / tots:4.1f}%  {k}")
