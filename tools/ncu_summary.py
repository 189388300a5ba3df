"""Text summary of an .ncu-rep (run here, no GPU needed): per kernel duration, DRAM bytes, pipe utilisation including
the tensor pipe, issue-slot use, plus the warp-stall breakdown and the hottest stall sites from the source page.
usage: python tools/ncu_summary.py x.ncu-rep > x.txt"""
import csv
import subprocess
import sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units, data = rows[0], rows[1], rows[2:]
KEYS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_op_hmma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_uniform.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "sm__cycles_active.avg", "sm__throughput.avg.pct_of_peak_sustained_elapsed"]
print(f"# ncu summary of {rep}  (ncu --set full --clock-control none; times are cold-cache, serialised replays)")
for r in data:
    print("\n== kernel:", r[hdr.index("Kernel Name")])
    for k in KEYS:
        if k in hdr:
            print(f"  {k:95s} {r[hdr.index(k)]:>18s} {units[hdr.index(k)]}")
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(src.splitlines()))
kern, cur = [], None
for r in rows:
    if r and r[0] == "Kernel Name":
        cur = {"name": r[1], "rows": []}
        kern.append(cur)
    elif cur is not None:
        cur["rows"].append(r)
seen = set()
for k in kern:
    if not k["rows"] or k["name"] in seen:
        continue
    h, d = k["rows"][0], k["rows"][1:]
    if "# Samples" not in h or "Source" not in h or not any("FFMA" in x[h.index("Source")] or "MUFU" in x[h.index("Source")] or "UTC" in x[h.index("Source")] for x in d):
        continue  # keep the SASS view only
    seen.add(k["name"])
    si, so = h.index("# Samples"), h.index("Source")
    sc = [i for i, x in enumerate(h) if x.startswith("stall_") and "Not Issued" not in x]
    tot = sum(int(r[si]) for r in d if r[si].isdigit()) or 1
    agg = {h[i]: sum(int(r[i]) for r in d if r[i].isdigit()) for i in sc}
    print(f"\n== warp-stall samples: {k['name']}  (total {tot})")
    print("  " + ", ".join(f"{a[6:]} {100 * b / tot:.1f}%" for a, b in sorted(agg.items(), key=lambda x: -x[1]) if b))
    top = sorted([(int(r[si]), i) for i, r in enumerate(d) if r[si].isdigit()], reverse=True)[:14]
    for n, i in sorted(top, key=lambda x: x[1]):
        r = d[i]
        st = {h[j][6:]: int(r[j]) for j in sc if r[j].isdigit() and int(r[j]) > 0}
        ctx = d[i - 1][so].strip()[:60] if "BRA" in r[so] else ""
        print(f"  {100 * n / tot:5.1f}%  {r[so].strip()[:58]:58s} {dict(sorted(st.items(), key=lambda x: -x[1])[:2])}  {ctx}")
