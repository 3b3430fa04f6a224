"""Condenses an ncu raw-page CSV (`ncu -i X.ncu-rep --page raw --csv > X.csv`, or a .ncu-rep directly when `ncu` is on PATH)
into the dozen numbers the design notes quote: duration, DRAM bytes and rate, instructions per work item, issue utilisation,
occupancy, lanes active per instruction, L2 hit rate, registers, top stall reasons.

    python tools/ncu_summary.py knn_thread_ncu_raw.csv [--items 1048576] [--alg-bytes 680]
"""
import csv
import io
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "dram read"),
    ("dram__bytes_write.sum", "dram write"),
    ("dram__bytes_read.sum.per_second", "dram read rate"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "dram throughput"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy"),
    ("smsp__thread_inst_executed_per_inst_executed.ratio", "lanes active / instruction"),
    ("launch__registers_per_thread", "registers / thread"),
    ("launch__shared_mem_per_block_static", "static smem / block"),
    ("launch__occupancy_limit_registers", "occupancy limit (registers, blocks)"),
    ("launch__occupancy_limit_shared_mem", "occupancy limit (smem, blocks)"),
]
UNIT = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "Tbyte": 1e12}


def load(path):
    if path.endswith(".ncu-rep"):
        txt = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    else:
        txt = open(path).read()
    rows = list(csv.reader(io.StringIO(txt)))
    hdr = rows[0]
    units = rows[1]
    return hdr, units, rows[2:]


def opt(name, default=None):
    return float(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def main():
    hdr, units, launches = load(sys.argv[1])
    items, alg = opt("--items"), opt("--alg-bytes")
    col = {h: i for i, h in enumerate(hdr)}
    name_i = col.get("Kernel Name")
    for r in launches:
        print("kernel:", r[name_i][:110], "| grid", r[col["Grid Size"]], "block", r[col["Block Size"]])
        vals = {}
        for key, label in KEYS:
            i = col.get(key)
            if i is None:
                continue
            vals[key] = (float(r[i].replace(",", "")) if r[i] not in ("", "n/a") else float("nan"), units[i])
            print(f"  {label:38s} {r[i]:>16s} {units[i]}")
        stalls = sorted(((float(r[i]), h.split("issue_stalled_")[1].split("_per_issue")[0]) for h, i in col.items()
                         if "smsp__average_warps_issue_stalled_" in h and h.endswith("_per_issue_active.ratio") and r[i] not in ("", "n/a")),
                        reverse=True)[:5]
        print("  top stalls (warps per issue):", ", ".join(f"{n} {v:.2f}" for v, n in stalls))
        if items:
            inst = vals.get("smsp__inst_executed.sum", (float("nan"), ""))[0]
            rd, ru = vals.get("dram__bytes_read.sum", (float("nan"), "byte"))
            dur, du = vals.get("gpu__time_duration.sum", (float("nan"), "us"))
            dur_s = dur * {"us": 1e-6, "ms": 1e-3, "ns": 1e-9, "s": 1.0}.get(du, 1e-6)
            print(f"  per item ({int(items)}): {inst / items:.1f} warp instructions, {rd * UNIT.get(ru, 1.0) / items:.0f} B of DRAM reads")
            if alg:
                print(f"  algorithmic: {alg:.0f} B/item -> {items * alg / dur_s / 1e9:.0f} GB/s")
        print()


if __name__ == "__main__":
    main()
