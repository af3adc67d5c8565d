"""Summarise an `ncu --set full ... --page raw --csv` export: one line per profiled launch with the numbers north_star asks for
(tensor-pipe % of peak for the contractions, achieved DRAM GB/s and % for the streams) plus duration, grid, registers, occupancy,
issue-slot use and L2 hit rate.
    python scripts/ncu_summary.py profiles/families_raw.csv > profiles/families_summary.txt"""
import csv, re, sys
rows = list(csv.reader(open(sys.argv[1])))
hdr, units, data = rows[0], rows[1], rows[2:]
col = {h: i for i, h in enumerate(hdr)}


def get(r, name, default=float("nan")):
    i = col.get(name)
    if i is None or i >= len(r) or r[i] in ("", "n/a"):
        return default
    try:
        return float(r[i].replace(",", ""))
    except ValueError:
        return default


def unit(name):
    return units[col[name]] if name in col else ""


def dur_us(r):
    v = get(r, "gpu__time_duration.sum")
    u = unit("gpu__time_duration.sum")
    return v / 1e3 if u in ("ns", "nsecond") else (v * 1e3 if u in ("ms", "msecond") else v)


def byts(r, name):
    v = get(r, name, 0.0)
    u = unit(name).lower()
    return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1)


print(f"# {sys.argv[1]}: ncu --set full, one line per launch; tensor% = sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active,")
print("# dram% = gpu__dram_throughput (avg % of peak), GB/s = (dram read + write) / duration, issue% = smsp__issue_active.avg.pct_of_peak_sustained_active, occ% = achieved occupancy")
print(f"{'kernel':46s} {'grid':>12s} {'blk':>5s} {'regs':>4s} {'us':>8s} {'tensor%':>8s} {'dram%':>6s} {'GB/s':>7s} {'rd MB':>8s} {'wr MB':>8s} {'L2hit%':>7s} {'issue%':>7s} {'occ%':>6s}")
for r in data:
    if len(r) < 10:
        continue
    name = re.sub(r"\(.*", "", r[col["Kernel Name"]]).replace("void ", "").replace("cgd::", "")
    us = dur_us(r)
    rd, wr = byts(r, "dram__bytes_read.sum"), byts(r, "dram__bytes_write.sum")
    tens = get(r, "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active")
    dram = get(r, "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed")
    l2 = get(r, "lts__t_sector_hit_rate.pct")
    issue = get(r, "smsp__issue_active.avg.pct_of_peak_sustained_active")
    occ = get(r, "sm__warps_active.avg.pct_of_peak_sustained_active")
    grid = r[col["Grid Size"]] if "Grid Size" in col else ""
    blk = r[col["Block Size"]] if "Block Size" in col else ""
    regs = get(r, "launch__registers_per_thread")
    gbs = (rd + wr) / (us * 1e-6) / 1e9 if us == us and us > 0 else float("nan")
    print(f"{name[:46]:46s} {grid.replace(' ', ''):>12s} {blk.replace(' ', '').replace(',1,1)', ')'):>5s} {regs:4.0f} {us:8.1f} {tens:8.1f} {dram:6.1f} {gbs:7.0f} {rd / 1e6:8.2f} {wr / 1e6:8.2f} {l2:7.1f} "
          f"{issue:7.1f} {occ:6.1f}")
