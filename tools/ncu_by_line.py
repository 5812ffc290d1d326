"""Attributes the SASS-level metrics of one kernel (ncu --page source --csv) to CUDA source lines.

usage:  cuobjdump -xelf all lib/libpb2.so; nvdisasm -g -c pb2_cuda.sm_90a.cubin > dis.txt
        ncu -i rep.ncu-rep --page source --csv > src.csv      (one kernel; cut the file if it holds several)
        python tools/ncu_by_line.py dis.txt src.csv <mangled-kernel-name-substring>
The disassembly and the profile must come from the same build: instructions are matched by position."""
import collections
import csv
import re
import sys

dis, src, key = sys.argv[1], sys.argv[2], sys.argv[3]
lines = open(dis).read().splitlines()
start = next(i for i, l in enumerate(lines) if l.startswith("\t.section\t.text.") and key in l)
loc = None
locs = []
for l in lines[start + 1:]:
    if l.startswith("\t.section") or l.startswith("//-----"):
        break
    m = re.search(r'//## File "([^"]+)", line (\d+)', l)
    if m:
        loc = (m.group(1).split("/")[-1], int(m.group(2)))
        continue
    if re.match(r"\s+/\*[0-9a-f]{4,}\*/\s", l):   # an instruction line: /*0010*/  OPCODE ...
        locs.append(loc)
rows = list(csv.reader(open(src)))
hdr = rows[1]
ci = {h: i for i, h in enumerate(hdr)}
body = rows[2:]
if len(body) != len(locs):
    print("warning: %d profiled instructions vs %d disassembled" % (len(body), len(locs)))
f = lambda x: float(x.replace(",", "") or 0)
inst = collections.Counter()
thr = collections.Counter()
smp = collections.Counter()
for r, lc in zip(body, locs):
    inst[lc] += f(r[ci["Instructions Executed"]])
    thr[lc] += f(r[ci["Thread Instructions Executed"]])
    smp[lc] += f(r[ci["# Samples"]])
ti, ts = sum(inst.values()), sum(smp.values())
print("kernel %s: %.0f warp instructions, %.0f samples" % (rows[0][1][:60], ti, ts))
srcs = {}
for (fn, ln), v in sorted(inst.items(), key=lambda kv: -(kv[1] / ti + smp[kv[0]] / max(ts, 1)))[:40] if ti else []:
    text = ""
    for root in ("pbrt_v3_b200/csrc/", "pbrt_v3_b200/csrc/device/"):
        try:
            srcs.setdefault(fn, open(root + fn).read().splitlines())
            text = srcs[fn][ln - 1].strip()[:90]
            break
        except Exception:
            pass
    print("%-22s %5d  instr %5.1f%%  samples %5.1f%%  thr %4.1f  %s" % (fn, ln, 100 * v / ti, 100 * smp[(fn, ln)] / max(ts, 1), thr[(fn, ln)] / max(v, 1), text))
