"""Per-kernel summary of an `ncu --set full` capture + the committed traffic table bench.py reads.

  python scripts/ncu_traffic.py X.ncu-rep --nodes 153600 --mode train --tag r03a [--out profiles/r03a_ncu_c1.txt]

Prints, per kernel name, the median launch: duration, DRAM bytes read / written, DRAM / L2 / SM throughput %, warps active,
tensor-pipe %, registers, grid; and updates profiles/ncu_traffic.json[kernel]["N=<nodes>,<mode>"] = {dram_read, dram_write,
duration_us, source} — `roofline.traffic` in bench.py is looked up there (never hard-coded)."""
import argparse
import csv
import io
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLS = {
    "dur_us": "gpu__time_duration.sum", "dram_rd": "dram__bytes_read.sum", "dram_wr": "dram__bytes_write.sum",
    "dram_pct": "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts_pct": "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm_pct": "sm__throughput.avg.pct_of_peak_sustained_elapsed", "warps_pct": "sm__warps_active.avg.pct_of_peak_sustained_active",
    "issue_pct": "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "tensor_pct": "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
    "regs": "launch__registers_per_thread", "grid": "launch__grid_size", "block": "launch__block_size",
    "st_sectors": "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
}
UNIT_SCALE = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "us": 1, "ms": 1e3, "ns": 1e-3, "s": 1e6, "usecond": 1, "msecond": 1e3, "nsecond": 1e-3}


def short(name):
    m = re.match(r"(?:void\s+)?((?:\w+::)*\w+)", name)
    return (m.group(1) if m else name).split("::")[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("rep")
    ap.add_argument("--nodes", type=int, required=True)
    ap.add_argument("--mode", default="train")
    ap.add_argument("--tag", required=True)
    ap.add_argument("--out")
    args = ap.parse_args()
    raw = subprocess.run(["ncu", "-i", args.rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    tensor_cols = [h for h in hdr if "tensor" in h and "cycles_active" in h and "pct" in h]
    by_kernel = {}
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        rec = {}
        for k, col in COLS.items():
            if k == "tensor_pct" and col not in d and tensor_cols:
                col = tensor_cols[0]
            if col in d and d[col] != "":
                try:
                    v = float(d[col].replace(",", ""))
                except ValueError:
                    continue
                rec[k] = v * UNIT_SCALE.get(units[hdr.index(col)], 1)
        by_kernel.setdefault(short(d["Kernel Name"]), []).append(rec)
    lines = [f"# {args.tag}: ncu --set full --clock-control none, median launch per kernel ({os.path.basename(args.rep)}; N = {args.nodes} nodes, {args.mode})"]
    table_path = os.path.join(ROOT, "profiles", "ncu_traffic.json")
    table = json.load(open(table_path)) if os.path.exists(table_path) else {}
    for name, recs in by_kernel.items():
        med = {k: statistics.median([r[k] for r in recs if k in r]) for k in COLS if any(k in r for r in recs)}
        tot = med.get("dram_rd", 0) + med.get("dram_wr", 0)
        gbs = tot / (med["dur_us"] * 1e-6) / 1e9 if med.get("dur_us") else 0
        lines.append(f"{name:32s} launches {len(recs):2d} | {med.get('dur_us', 0):8.1f} us | DRAM rd {med.get('dram_rd', 0) / 1e6:8.1f} MB wr {med.get('dram_wr', 0) / 1e6:8.1f} MB "
                     f"= {gbs:6.0f} GB/s | dram {med.get('dram_pct', 0):5.1f}% l2 {med.get('lts_pct', 0):5.1f}% sm {med.get('sm_pct', 0):5.1f}% | warps {med.get('warps_pct', 0):5.1f}% "
                     f"issue {med.get('issue_pct', 0):5.1f}% tensor {med.get('tensor_pct', 0):5.1f}% | regs {int(med.get('regs', 0))} grid {int(med.get('grid', 0))}x{int(med.get('block', 0))} "
                     f"| st sectors {med.get('st_sectors', 0) / 1e6:6.2f} M")
        table.setdefault(name, {})[f"N={args.nodes},{args.mode}"] = {
            "dram_read": int(med.get("dram_rd", 0)), "dram_write": int(med.get("dram_wr", 0)), "duration_us": round(med.get("dur_us", 0), 2),
            "launches": len(recs), "source": f"profiles/{os.path.basename(args.out) if args.out else args.tag}"}
    text = "\n".join(lines)
    print(text)
    if args.out:
        open(args.out, "w").write(text + "\n")
    json.dump(table, open(table_path, "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
