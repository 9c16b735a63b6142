"""Per-source-line dynamic instruction profile of the NUTS kernel from an `ncu --page source --csv` export (SASS view with
executed counts) joined with `nvdisasm -c -gi` line / inline info of the SAME build.
Usage: python scripts/ncu_line_profile.py <source.csv> <nvdisasm -gi listing of the kernel> <kernel .cu> <device .cuh> <leaves> [inner]
("inner": attribute to the INNERMOST frame inside the kernel's own file instead of the outermost -- for kernels whose
 body is one big inlined call, e.g. K4's tile product)"""
import collections
import csv
import re
import sys

csv.field_size_limit(10 ** 9)
path_csv, path_sass, path_cu, path_dev, leaves = sys.argv[1], sys.argv[2], sys.argv[3], sys.argv[4], float(sys.argv[5])
inner_mode = len(sys.argv) > 6 and sys.argv[6] == "inner"
rows = list(csv.reader(open(path_csv)))
starts = [i for i, r in enumerate(rows) if len(r) > 5 and r[0] == "Address" and "Source" in r]
s = starts[0]  # first table = first captured launch
hdr = rows[s]
body = [r for r in rows[s + 1:(starts[1] if len(starts) > 1 else len(rows))] if len(r) == len(hdr)]
ix = {n: i for i, n in enumerate(hdr)}
ex = [float(r[ix["Instructions Executed"]] or 0) for r in body]
samp = [float(r[ix["# Samples"]] or 0) for r in body]
cu_name = path_cu.split("/")[-1]
dev_name = path_dev.split("/")[-1]
ann, pending, cur = [], [], None
for ln in open(path_sass).read().splitlines():
    m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
    if m:
        pending.append((m.group(1).split("/")[-1], int(m.group(2))))
        continue
    if re.match(r"\s*/\*[0-9a-f]+\*/\s+\S", ln):
        if pending:
            own = [q for q in pending if q[0] == cu_name]
            kline = (own[0][1] if own else None) if inner_mode else (pending[-1][1] if pending[-1][0] == cu_name else None)
            cur = (kline, pending[0])
            pending = []
        ann.append(cur)
assert len(ann) == len(ex), (len(ann), len(ex))
src, dev = open(path_cu).read().splitlines(), open(path_dev).read().splitlines()


def func_of(lines, l):
    for i in range(l - 1, -1, -1):
        m = re.search(r"(?:__device__|__global__)[^;{]*?\b([A-Za-z_0-9]+)\s*\(", lines[i])
        if m and not lines[i].strip().startswith("//"):
            return m.group(1)
    return "?"


tot, tots = sum(ex), sum(samp)
byk, byks, byf, byfs = (collections.Counter() for _ in range(4))
stall_cols = [n for n in hdr if n.startswith("stall_") and "Not Issued" not in n]
why = collections.defaultdict(collections.Counter)
for c, e, sm, r in zip(ann, ex, samp, body):
    if c is None:
        continue
    for n in stall_cols:
        why[c[0]][n[6:]] += float(r[ix[n]] or 0)
    kl, inner = c
    byk[kl] += e
    byks[kl] += sm
    fn = func_of(dev, inner[1]) if inner[0] == dev_name else ("[kernel body / libdevice]" if inner[0] == cu_name else inner[0])
    byf[fn] += e
    byfs[fn] += sm
print(f"{tot:.0f} warp-instructions over {leaves:.0f} leaves = {tot / leaves:.0f} per leaf; {tots:.0f} stall samples")
print("\ninnermost function: warp-instructions per leaf | % of instructions | % of stall samples")
for fn, e in byf.most_common(18):
    print(f"  {fn:28s} {e / leaves:7.1f} {100 * e / tot:6.1f}% {100 * byfs[fn] / tots:6.1f}%")
print(f"\nkernel source line ({'innermost' if inner_mode else 'outermost'} frame in {cu_name}): per leaf | % instr | % stalls | top stall reasons | source")
order = sorted(byk, key=lambda k: -(byks[k] if inner_mode else byk[k]))[:32]
for kl in order:
    e = byk[kl]
    top = ", ".join(f"{k}:{v:.0f}" for k, v in why[kl].most_common(2))
    print(f"  L{kl}: {e / leaves:8.1f} {100 * e / tot:5.1f}% {100 * byks[kl] / tots:5.1f}%  [{top}]  {src[kl - 1].strip()[:100] if kl else ''}")
