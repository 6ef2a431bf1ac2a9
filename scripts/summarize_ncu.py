"""Turn ncu artefacts (a launch-list CSV or a kernel report) into text summaries on stdout.

  python scripts/summarize_ncu.py launches launches.csv
  python scripts/summarize_ncu.py kernel xpbd.ncu-rep
"""
import collections, csv, subprocess, sys

def launches(path):
    rows = list(csv.reader(open(path)))
    hdr, agg = None, collections.defaultdict(lambda: [0, 0.0])
    for r in rows:
        if len(r) > 5 and r[0] == "ID":
            hdr = r
            continue
        if hdr and len(r) == len(hdr):
            name = r[4].split("(")[0][:70]
            agg[name][0] += 1
            agg[name][1] += float(r[-1])
    tot = sum(v[1] for v in agg.values())
    print(f"# ncu --metrics gpu__time_duration.sum --clock-control none (cold-cache, serialised: compare SHARES) : {path}")
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{k:72s} n={v[0]:4d} total_us={v[1]/1e3:10.1f} share={v[1]/tot*100:5.1f}% avg_us={v[1]/v[0]/1e3:8.1f}")

WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__warps_active.avg.per_cycle_active",
        "smsp__warps_eligible.avg.per_cycle_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_blocks", "launch__grid_size", "launch__block_size",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed.sum"]

def kernel(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr = rows[0]
    print(f"# ncu --set full --clock-control none --import-source on : {path}")
    ki = hdr.index("Kernel Name")
    print("kernel:", rows[2][ki][:120])
    for w in WANT:
        if w in hdr:
            i = hdr.index(w)
            print(f"{w:70s} {[r[i] for r in rows[2:]]} {rows[1][i]}")
    sass = subprocess.run(["ncu", "-i", path, "--page", "source", "--csv", "--print-source", "sass"], capture_output=True, text=True).stdout
    rows = list(csv.reader(sass.splitlines()))
    nk = sum(1 for r in rows if r and r[0] == "Kernel Name")
    hdr = rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    data = [r for r in rows[2:] if len(r) == len(hdr) and r[0] != "Address"]
    data = data[: len(data) // max(nk, 1)]
    def f(r, k):
        try:
            return float(r[idx[k]])
        except Exception:
            return 0.0
    tot = sum(f(r, "Instructions Executed") for r in data)
    print(f"static SASS instructions: {len(data)}   warp-instructions executed: {tot:.0f}")
    stalls = [h for h in hdr if h.startswith("stall_") and "Not Issued" not in h]
    agg = {s: sum(f(r, s) for r in data) for s in stalls}
    ts = sum(agg.values()) or 1.0
    print("warp stall sampling (all samples):")
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1])[:10]:
        print(f"  {k:28s} {v:9.0f} {v/ts*100:5.1f}%")
    op = collections.Counter()
    for r in data:
        s = r[idx["Source"]].split()
        if not s:
            continue
        o = s[0] if not s[0].startswith("@") else (s[1] if len(s) > 1 else s[0])
        op[o.split(".")[0]] += f(r, "Instructions Executed")
    print("opcode mix (executed warp-instructions):")
    for k, v in op.most_common(14):
        print(f"  {k:10s} {v:12.0f} {v/tot*100:5.1f}%")

if __name__ == "__main__":
    {"launches": launches, "kernel": kernel}[sys.argv[1]](sys.argv[2])
