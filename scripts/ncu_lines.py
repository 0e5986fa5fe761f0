"""Per-source-line instruction / stall profile of one kernel from an ncu report.

  python scripts/ncu_lines.py gpurun_out/prof.ncu-rep [kernel-symbol-substring] [rows]
  (NCU_LINES_UNIT=runs_tma picks frostdb_b200/csrc/runs_tma.cu / build/runs_tma.o instead of kernels)

Joins `ncu --page source --csv` (per-SASS-instruction counters, in program order) with
`nvdisasm -g` of the cubin inside frostdb_b200/csrc/build/kernels.o (line markers, same order)."""
import collections, csv, io, os, re, subprocess, sys, tempfile

rep = sys.argv[1]
sym = sys.argv[2] if len(sys.argv) > 2 else "k_scan"
rows_scanned = float(sys.argv[3]) if len(sys.argv) > 3 else 0
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
csrc = os.path.join(root, "frostdb_b200", "csrc")
unit = os.environ.get("NCU_LINES_UNIT", "kernels")
tmp = tempfile.mkdtemp()
subprocess.check_call(["cuobjdump", "-xelf", "all", os.path.join(csrc, "build", unit + ".o")], cwd=tmp, stdout=subprocess.DEVNULL)
dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(tmp, f"{unit}.sm_90a.cubin")], capture_output=True, text=True).stdout
cur_fn, cur_line, seq = None, None, []
for ln in dis.split("\n"):
    if ln.startswith("\t.section") and ".text." in ln:
        cur_fn, cur_line = ln.split(".text.")[1].split(",")[0], None
        continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
    if m:
        cur_line = (os.path.basename(m.group(1)), int(m.group(2)))
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", ln)
    if m and cur_fn and sym in cur_fn:
        seq.append((cur_line, m.group(2).strip()))
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(out)))
hdr = rows[1]
ix = {h: i for i, h in enumerate(hdr)}
data = [r for r in rows[2:] if len(r) == len(hdr)]
assert len(data) == len(seq), (len(data), len(seq), "rebuild kernels.o at the profiled commit")


def f(r, k):
    try:
        return float(r[ix[k]])
    except Exception:
        return 0.0


inst, samp = collections.Counter(), collections.Counter()
stall = collections.Counter()
for (line, _), r in zip(seq, data):
    inst[line] += f(r, "Instructions Executed")
    samp[line] += f(r, "# Samples")
    for h in hdr:
        if h.startswith("stall_") and "Not" not in h:
            stall[h] += f(r, h)
ti, ts = sum(inst.values()), sum(samp.values())
print(f"warp instructions {ti:.0f}" + (f"  = {ti / (rows_scanned / 32):.1f} per 32-row step" if rows_scanned else ""))
ss = sum(stall.values())
print("stalls:", ", ".join(f"{k[6:]} {v / ss * 100:.0f}%" for k, v in stall.most_common(7)))
src = open(os.path.join(csrc, unit + ".cu")).read().split("\n")
# per function (source ranges between "__device__"/"__global__" definitions)
starts = [i + 1 for i, l in enumerate(src) if re.match(r"^(template .*)?(__device__|__global__)", l) or (l.startswith("__device__") or l.startswith("__global__"))]
def fn_of(line):
    best = 0
    for s in starts:
        if s <= line:
            best = s
    return src[best - 1].strip()[:90] if best else "?"
byfn_i, byfn_s = collections.Counter(), collections.Counter()
for k, v in inst.items():
    name = fn_of(k[1]) if k and k[0] == unit + ".cu" else (k[0] if k else "?")
    byfn_i[name] += v
    byfn_s[name] += samp[k]
print("\n-- by function: inst%  samples%")
for name, v in byfn_i.most_common(22):
    print(f"{v / ti * 100:5.1f} {byfn_s[name] / ts * 100:5.1f}  {name}")
print("\n-- by line: inst%  samples%")
for k, v in inst.most_common(int(os.environ.get("NCU_LINES_TOP", 40))):
    if not k:
        continue
    text = src[k[1] - 1].strip()[:100] if k[0] == unit + ".cu" else k[0]
    print(f"{k[1]:5d} {v / ti * 100:5.1f} {samp[k] / ts * 100:5.1f}  {text}")
